"""Times derp_gaussian_blur (include/derp_b200.h) and GenerateForegroundMasks on one GPU and writes one JSON file.

  blur     : derp_gaussian_blur of a 2048 x 1024 u16 x 3 image (the app's default --width) at radii 1, 2, 3, 4 and 20,
             timed with CUDA events over --reps calls after a warm-up call, on device-resident buffers and on pageable
             host buffers as the app passes them (the staging copies are inside that window)
  host     : the host blur GenerateForegroundMasks ran at radii 2 and 3 before (io::gaussianBlurU16C3, through IoSelfTest
             --mode=gauss): wall time of the process, which includes its start and the raw read and write of the image
  app      : GenerateForegroundMasks on the golden 16-camera rig (tests/golden/sweep_rig16.json, 3360 x 2160 16-bit PNG
             backgrounds and frames, one frame, --width 2048) at --blur_radius 1, 2 and 20: wall time of the process, two
             runs each after one warm-up run
Usage: python tools/foreground_mask_bench.py [--out profiles/h100_foreground_masks_16cam.json] [--reps 20]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from facebook360_dep_b200 import capi  # noqa: E402

BIN = os.path.join(ROOT, "facebook360_dep_b200", "bin")
GOLDEN_RIG = os.path.join(ROOT, "tests", "golden", "sweep_rig16.json")
W, H = 2048, 1024


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    name, limit = [s.strip() for s in out.split(",")]
    return name, limit


def time_call(fn, reps):
    fn()  # warm-up
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return ms


def wall(cmd):
    t0 = time.perf_counter()
    p = subprocess.run(cmd, capture_output=True, text=True)
    dt = time.perf_counter() - t0
    assert p.returncode == 0, p.stderr[-2000:]
    return dt


def write_rig_frames(tmp, rig):
    """A smooth background per camera and a frame with a textured foreground patch, as 16-bit PNG files."""
    import cv2
    rng = np.random.RandomState(0)
    for s, cam in enumerate(rig["cameras"]):
        w, h = cam["resolution"]
        yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
        bg = np.stack([20000 + 8000 * np.sin(xx / (300 + 20 * s)), 30000 + 6000 * np.cos(yy / 250),
                       25000 + 4000 * np.sin((xx + yy) / 400)], -1)
        fr = bg.copy()
        fr[h // 4:h // 2, w // 3:w // 3 + 600] += rng.randint(-12000, 12000, (h // 2 - h // 4, 600, 3))
        for d, img, frame in (("bg", bg, "000000"), ("fg", fr, "000001")):
            os.makedirs(os.path.join(tmp, d, cam["id"]), exist_ok=True)
            cv2.imwrite(os.path.join(tmp, d, cam["id"], frame + ".png"), np.clip(img, 0, 65535).astype(np.uint16))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_foreground_masks_16cam.json"))
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no GPU: nothing is measured")
    gpu, limit = gpu_info()
    lib = capi.Blur(capi.load_cuda())
    img = np.random.RandomState(1).randint(0, 65536, (H, W, 3)).astype(np.uint16)
    out = np.empty_like(img)
    dsrc = torch.from_numpy(img).cuda()
    ddst = torch.empty_like(dsrc)
    result = dict(workload="derp_gaussian_blur at 2048 x 1024 u16 x 3; GenerateForegroundMasks on the golden 16-camera "
                           "rig (3360 x 2160 PNG, --width 2048, one frame)", gpu=gpu, power_limit=limit, reps=args.reps,
                  blur={}, host_blur={}, app={})
    for r in (1, 2, 3, 4, 20):
        dev = time_call(lambda: lib.check(lib.lib.derp_gaussian_blur(0, dsrc.data_ptr(), W, H, r, ddst.data_ptr())), args.reps)
        host = time_call(lambda: lib.check(lib.lib.derp_gaussian_blur(0, img.ctypes.data, W, H, r, out.ctypes.data)), args.reps)
        result["blur"][str(r)] = dict(device_ms=dev, device_ms_median=float(np.median(dev)), host_ms=host,
                                      host_ms_median=float(np.median(host)))
    with tempfile.TemporaryDirectory() as tmp:
        raw, blurred = os.path.join(tmp, "img.raw"), os.path.join(tmp, "img.out")
        img.tofile(raw)
        for r in (2, 3):
            cmd = [os.path.join(BIN, "IoSelfTest"), "--mode=gauss", "--in=" + raw, "--width=%d" % W, "--height=%d" % H,
                   "--size=%d" % r, "--out=" + blurred]
            wall(cmd)  # warm the page cache
            s = [wall(cmd) for _ in range(3)]
            result["host_blur"][str(r)] = dict(wall_s=s, wall_s_median=float(np.median(s)))
            assert np.array_equal(np.fromfile(blurred, np.uint16).reshape(H, W, 3),
                                  lib.gaussian_blur(img, r)), r
        rig = json.load(open(GOLDEN_RIG))
        write_rig_frames(tmp, rig)
        for r in (1, 2, 20):
            cmd = [os.path.join(BIN, "GenerateForegroundMasks"), "--rig=" + GOLDEN_RIG, "--color=" + os.path.join(tmp, "fg"),
                   "--background_color=" + os.path.join(tmp, "bg"), "--foreground_masks=" + os.path.join(tmp, "m%d" % r),
                   "--first=000001", "--last=000001", "--blur_radius=%d" % r]
            if r == 1:
                wall(cmd)  # warm-up: the page cache of the PNG files
            s = [wall(cmd) for _ in range(2)]
            result["app"][str(r)] = dict(wall_s=s, wall_s_median=float(np.median(s)), cameras=len(rig["cameras"]))
    line = json.dumps(result)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
