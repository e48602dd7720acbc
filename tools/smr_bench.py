#!/usr/bin/env python3
"""Time SimpleMeshRenderer per format on the GPU: a 16-camera FTHETA ring, disparity 1024^2, colour 2048^2, --width 3072
(equirect and cube edge 1536, snapshot 3072 x 1536).

Prints one JSON line.  Per format: the wall time of one app run on one frame (process start, loading, rendering,
compositing and the png write), and the device time of the same renders through the binding, summed per stage from a
torch.profiler CUDA trace: prep (mesh, textures, mips), raster (depth / primitive bids), resolve (shading, blend,
unpremultiply) and equirect (the cube to equirect resample).  The GPU's name and power limit are read in the same run.
Inputs and outputs go to a temporary directory; nothing is written in the tree unless --out is given."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

from facebook360_dep_b200 import capi, synth  # noqa: E402
from tools.wide_rig_bench import gpu_conditions  # noqa: E402

STAGES = {"prep": ("rephotoPrepKernel", "rephotoMipKernel"), "raster": ("rephotoRasterKernel",),
          "resolve": ("rephotoResolveKernel", "rephotoUnpremulKernel"), "equirect": ("canopyEquirectKernel",)}
FORMATS = ["cubecolor", "cubedisp", "eqrcolor", "eqrdisp", "lr180", "snapcolor", "snapdisp", "tb3dof", "tbstereo"]


def renders(lib, descs, disps, bgra, fmt, width):
    """The derp_canopy_render calls the app makes for one frame of `fmt`."""
    h = width // 2
    pos = np.zeros(3, np.float32)
    disp = fmt in ("cubedisp", "eqrdisp", "snapdisp")
    kw = dict(want_color=not disp, want_disparity=disp)
    if fmt.startswith("cube"):
        lib.render(descs, disps, bgra, pos, "cubemap", (h, h), **kw)
    elif fmt.startswith("eqr"):
        lib.render(descs, disps, bgra, pos, "equirect", (2 * h, h), **kw)
    elif fmt.startswith("snap"):
        m = capi.snapshot_matrix(pos, [-1, 0, 0], [0, 0, 1], 90.0, width, h)
        lib.render(descs, disps, bgra, pos, "perspective", (width, h), m, **kw)
    elif fmt == "tb3dof":
        lib.render(descs, disps, bgra, pos, "equirect", (2 * h, h))
        lib.render(descs, disps, bgra, pos, "equirect", (2 * h, h), want_color=False, want_disparity=True)
    else:
        for ipd in (0.032, -0.032):
            lib.render(descs, disps, bgra, pos, "equirect", (2 * h, h), ipd=ipd)


def stage_ms(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        events = json.load(open(path)).get("traceEvents", [])
    out = {k: 0.0 for k in STAGES}
    for e in events:
        if e.get("cat") != "kernel":
            continue
        for k, names in STAGES.items():
            if any(n in e.get("name", "") for n in names):
                out[k] += e.get("dur", 0) / 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cams", type=int, default=16)
    ap.add_argument("--disparity", type=int, default=1024)
    ap.add_argument("--color", type=int, default=2048)
    ap.add_argument("--width", type=int, default=3072)
    ap.add_argument("--formats", default=",".join(FORMATS))
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    lib = capi.Canopy(capi.load_cuda())
    D, Cs = a.disparity, a.color
    rig = synth.ring_rig(a.cams, Cs, Cs, kind="FTHETA")
    colors, gt = synth.render_rig(rig, Cs, Cs, device="cuda")
    step = Cs // D
    disps = [np.ascontiguousarray(d[::step, ::step]) for d in gt]
    bgra = [np.concatenate([c.astype(np.float32) * np.float32(1 / 65535), np.ones((Cs, Cs, 1), np.float32)], -1)
            for c in colors]
    descs = capi.rig_descs(rig)
    result = {"tool": "tools/smr_bench.py", "gpu": gpu_conditions(),
              "config": {"cameras": a.cams, "camera_model": "FTHETA ring", "disparity": D, "color": Cs,
                         "width": a.width, "shader": "canopyFS_SVD", "alpha_blend": True},
              "formats": {}}
    app = os.path.join(capi.ROOT, "facebook360_dep_b200", "bin", "SimpleMeshRenderer")
    with tempfile.TemporaryDirectory() as tmp:
        json.dump(rig, open(os.path.join(tmp, "rig.json"), "w"))
        for cam, c, d in zip(rig["cameras"], colors, disps):
            for sub in ("color", "disparity"):
                os.makedirs(os.path.join(tmp, sub, cam["id"]), exist_ok=True)
            assert cv2.imwrite(os.path.join(tmp, "color", cam["id"], "000000.png"), c)
            with open(os.path.join(tmp, "disparity", cam["id"], "000000.pfm"), "wb") as f:
                f.write(b"Pf\n%d %d\n-1.0\n" % (D, D))
                f.write(np.ascontiguousarray(d, np.float32).tobytes())  # this project's PFM: top row first
        renders(lib, descs, disps, bgra, "tb3dof", a.width)  # warm-up: module load, scratch allocation
        for fmt in a.formats.split(","):
            t0 = time.perf_counter()
            subprocess.run([app, "--rig=" + os.path.join(tmp, "rig.json"), "--color=" + os.path.join(tmp, "color"),
                            "--disparity=" + os.path.join(tmp, "disparity"), "--output=" + os.path.join(tmp, fmt),
                            "--format=" + fmt, "--width=%d" % a.width], check=True, capture_output=True)
            wall = (time.perf_counter() - t0) * 1e3
            dev = stage_ms(lambda: renders(lib, descs, disps, bgra, fmt, a.width))
            result["formats"][fmt] = {"app_wall_ms": wall, "device_ms": sum(dev.values()), "stage_device_ms": dev}
    line = json.dumps(result, ensure_ascii=False)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
