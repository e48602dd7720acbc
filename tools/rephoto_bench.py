#!/usr/bin/env python3
"""Time ComputeRephotographyErrors' per-camera work on the GPU: for one camera of a 16-camera FTHETA ring, the reference
cubemap (its own canopy), the rendered cubemap (the other 15 canopies), both with their disparity cubemaps, and the
MSSIM score — what the app does per camera and frame.  Sizes 1024^2 and 2048^2 (cube edge = image height).

Prints one JSON line: wall time per camera (host clock around the synchronous entry points, inputs in host memory as
the app passes them), and the device time of each stage summed from a torch.profiler CUDA trace of one more camera:
canopy preparation (mesh, RGBA16 texture, mips), raster (depth / primitive bids), accumulate (resolve, shading, blend,
unpremultiply) and score (Gaussian blurs, SSIM, masked sums).  The GPU's name and power limit are read in the same run.
Writes nothing in the tree unless --out is given."""
import argparse
import json
import os
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from facebook360_dep_b200 import capi, synth  # noqa: E402
from tools.wide_rig_bench import gpu_conditions  # noqa: E402

STAGES = {"prepare": ("rephotoPrepKernel", "rephotoMipKernel"), "raster": ("rephotoRasterKernel",),
          "accumulate": ("rephotoResolveKernel", "rephotoUnpremulKernel"),
          "score": ("rephotoBlurRowsKernel", "rephotoBlurColsKernel", "rephotoMomentsKernel", "rephotoScoreKernel")}


def one_camera(lib, rig, disps, bgra, i):
    cams = rig["cameras"]
    W = disps[0].shape[0]
    ctr = np.array(cams[i]["origin"], np.float32)
    others = [j for j in range(len(cams)) if j != i]
    ref = lib.rephoto_cubemap(capi.rig_descs({"cameras": [cams[i]]}), [disps[i]], [bgra[i]], ctr, W, want_disparity=True)
    ren = lib.rephoto_cubemap(capi.rig_descs({"cameras": [cams[j] for j in others]}), [disps[j] for j in others],
                              [bgra[j] for j in others], ctr, W, want_disparity=True)
    mask = (ref[0][..., 3] > 0).astype(np.uint8)
    return lib.rephoto_score(ref[0][..., :3], ren[0][..., :3], mask, "MSSIM", 1)[1]


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
    ap.add_argument("--sizes", default="1024,2048")
    ap.add_argument("--cams", type=int, default=16)
    ap.add_argument("--timed", type=int, default=2, help="cameras timed per size (after one warm-up camera)")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    lib = capi.Rephoto(capi.load_cuda())
    result = {"tool": "tools/rephoto_bench.py", "gpu": gpu_conditions(),
              "config": {"cameras": a.cams, "camera_model": "FTHETA ring", "method": "MSSIM", "stat_radius": 1,
                         "timed": "per camera: 2 x derp_rephoto_cubemap (colour + disparity) + derp_rephoto_score"},
              "sizes": {}}
    for W in (int(s) for s in a.sizes.split(",")):
        rig = synth.ring_rig(a.cams, W, W, kind="FTHETA")
        colors, disps = synth.render_rig(rig, W, W, device="cuda")
        bgra = [np.concatenate([c.astype(np.float32) * np.float32(1 / 65535), np.ones((W, W, 1), np.float32)], -1)
                for c in colors]
        one_camera(lib, rig, disps, bgra, 0)  # warm-up: module load, scratch allocation
        times, scores = [], []
        for i in range(1, 1 + a.timed):
            t0 = time.perf_counter()
            scores.append(one_camera(lib, rig, disps, bgra, i).tolist())
            times.append((time.perf_counter() - t0) * 1e3)
        result["sizes"][str(W)] = {"ms_per_camera": float(np.mean(times)), "ms_per_camera_runs": times,
                                   "stage_device_ms": stage_ms(lambda: one_camera(lib, rig, disps, bgra, a.timed + 1)),
                                   "mssim_bgr": scores}
    line = json.dumps(result, ensure_ascii=False)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
