"""Times derp_resize_area (include/derp_resize.h) and ResizeFrames on one GPU against resize.py's cv2 work, and writes one
JSON file.  The workload is the golden 16-camera rig (tests/golden/sweep_rig16.json, 3360 x 2160): 16-bit 3-channel
colour and 8-bit 1-channel foreground masks (0 / 255, resized with --threshold 127).

  library : the ten levels of one 3360 x 2160 image (ten derp_resize_area calls), timed with CUDA events over --reps
            repetitions after a warm-up, from a device-resident source into device buffers, and from pageable host memory
            into pageable host memory (the staging copies are inside that window)
  app     : ResizeFrames on one frame of the 16 cameras (colour, then masks): wall time of the process, two runs each
            after a warm-up run
  cv2     : resize_camera's per-image work (resize.py:51-85: cv2.imread(UNCHANGED), ten cv2.resize(INTER_AREA)
            [+ cv2.threshold], ten cv2.imwrite) on one camera, in this process on this host, --reps times
  png     : the share of that cv2 work spent in imread and imwrite, to show what bounds the app
Usage: python tools/resize_frames_bench.py [--out profiles/h100_resize_frames_16cam.json] [--reps 10]"""
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
WIDTHS = [2048, 1024, 512, 256, 200, 128, 100, 80, 60, 50]
SW, SH = 3360, 2160


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    name, limit = [s.strip() for s in out.split(",")]
    return name, limit


def levels():
    out = []
    for w in WIDTHS:
        h = round(SH / SW * w)
        out.append((w, h + h % 2))
    return out


def time_events(fn, reps):
    fn()
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


def images(kind, seed):
    """Smooth colour with texture (16-bit x 3) or a blob mask (8-bit, 0 / 255): content that compresses like a frame."""
    rng = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:SH, 0:SW].astype(np.float32)
    if kind == "color":
        img = np.stack([20000 + 8000 * np.sin(xx / (300 + 20 * seed)), 30000 + 6000 * np.cos(yy / 250),
                        25000 + 4000 * np.sin((xx + yy) / 400)], -1) + rng.randint(-500, 500, (SH, SW, 3))
        return np.clip(img, 0, 65535).astype(np.uint16)
    return ((((xx - SW / 2 - 40 * seed) / 900) ** 2 + ((yy - SH / 2) / 600) ** 2) < 1).astype(np.uint8) * 255


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_resize_frames_16cam.json"))
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no GPU: nothing is measured")
    import cv2
    gpu, limit = gpu_info()
    lib = capi.Resize(capi.load_cuda())
    rig = json.load(open(GOLDEN_RIG))
    result = dict(workload="pyramid resize of the golden 16-camera rig (3360 x 2160) to the ten widths of config.WIDTHS: "
                           "16-bit 3-channel colour and 8-bit 1-channel masks (--threshold 127)", gpu=gpu,
                  power_limit=limit, reps=args.reps, cv2_version=cv2.__version__, cv2_threads=cv2.getNumThreads(),
                  library={}, app={}, cv2={})
    with tempfile.TemporaryDirectory() as tmp:
        for kind, bits, ch, thr in (("color", 16, 3, -1), ("masks", 8, 1, 127)):
            img = images(kind, 0)
            outs = [np.empty((h, w) + img.shape[2:], img.dtype) for w, h in levels()]
            dsrc = torch.from_numpy(img).cuda()
            douts = [torch.from_numpy(o).cuda() for o in outs]

            def device_levels():
                for (w, h), o in zip(levels(), douts):
                    lib.check(lib.lib.derp_resize_area(0, dsrc.data_ptr(), bits, ch, SW, SH, o.data_ptr(), w, h, thr))

            def host_levels():
                for (w, h), o in zip(levels(), outs):
                    lib.check(lib.lib.derp_resize_area(0, img.ctypes.data, bits, ch, SW, SH, o.ctypes.data, w, h, thr))

            dev, host = time_events(device_levels, args.reps), time_events(host_levels, args.reps)
            result["library"][kind] = dict(device_ms=dev, device_ms_median=float(np.median(dev)), host_ms=host,
                                           host_ms_median=float(np.median(host)))
            src = os.path.join(tmp, kind)
            for s, cam in enumerate(rig["cameras"]):
                os.makedirs(os.path.join(src, cam["id"]))
                cv2.imwrite(os.path.join(src, cam["id"], "000000.png"), images(kind, s))
            cmd = [os.path.join(BIN, "ResizeFrames"), "--rig=" + GOLDEN_RIG, "--src_dir=" + src,
                   "--dst_dir=" + os.path.join(tmp, kind + "_levels"), "--threshold=%d" % thr]
            wall(cmd)  # warm-up: the page cache of the PNG files
            s = [wall(cmd) for _ in range(2)]
            result["app"][kind] = dict(wall_s=s, wall_s_median=float(np.median(s)), images=len(rig["cameras"]))
            # resize_camera on one camera, in this process
            path = os.path.join(src, rig["cameras"][0]["id"], "000000.png")
            total, io_s = [], []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                im = cv2.imread(path, cv2.IMREAD_UNCHANGED)
                t_io = time.perf_counter() - t0
                for level, (w, h) in enumerate(levels()):
                    scaled = cv2.resize(im, (w, h), interpolation=cv2.INTER_AREA)
                    if thr >= 0:
                        _, scaled = cv2.threshold(scaled, thr, 255, cv2.THRESH_BINARY)
                    t1 = time.perf_counter()
                    cv2.imwrite(os.path.join(tmp, "cv_%d.png" % level), scaled)
                    t_io += time.perf_counter() - t1
                total.append(time.perf_counter() - t0)
                io_s.append(t_io)
            result["cv2"][kind] = dict(per_image_s=total, per_image_s_median=float(np.median(total)),
                                       png_s_median=float(np.median(io_s)))
    line = json.dumps(result)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
