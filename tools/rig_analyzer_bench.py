"""Times RigAnalyzer's coverage counts (include/derp_riganalysis.h) and app on one GPU, on the golden 16-camera FTHETA
rig (tests/golden/sweep_rig16.json, 3360 x 2160) at the app's defaults, and writes one JSON file.

  entry points : derp_rig_coverage (100 000 samples x 20 distances), derp_rig_equirect_coverage (1800 x 900 with the
                 timing plane), derp_rig_camera_coverage (camera cam0, 3360 x 2160) and derp_rig_cross_section
                 (400 x 400), each at --overlap_distance 1e4, timed with CUDA events over --reps calls after a warm-up
                 call (host outputs: the copy back is inside the window), with the share of points the host resolved
  app          : RigAnalyzer --output_obj --output_equirect --output_camera (cam0) --output_cross_section, wall time of
                 the process; "host" is that wall time minus the four entry points' medians (process start, rig
                 loading, the report and the text files)
  cpu          : the checker's main (the reference's own RigAnalyzer.cpp, oracle/riganalyzer.mk) with the same flags,
                 on one host thread as the reference runs
Usage: python tools/rig_analyzer_bench.py [--out profiles/h100_rig_analyzer_16cam.json] [--reps 5] [--no-cpu]"""
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
from tests import riganalyzer_util as ru  # noqa: E402


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_rig_analyzer_16cam.json"))
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-cpu", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no GPU: nothing is measured")
    gpu, limit = gpu_info()
    lib = capi.RigAnalysis(capi.load_cuda())
    d = ru.descs_of(ru.GOLDEN_RIG)
    # getFibonacciUnits(100000) as the app computes it (discard_poles 0 keeps every sample)
    i = np.arange(100000)
    y = (i + 0.5) / 100000 * 2 - 1
    r = np.sqrt(1 - y * y)
    roty = i / ((1 + np.sqrt(5)) / 2) * 2 * np.pi
    samples = np.stack([np.sin(roty) * r, y, np.cos(roty) * r], 1)
    dists = [0.5 / (1 - k / 20.0) for k in range(20)]
    calls = {
        "coverage": (lambda: lib.coverage(d, samples, dists), len(samples) * len(dists)),
        "equirect": (lambda: lib.equirect(d, 1800, 900, 1e4), 1800 * 900),
        "camera": (lambda: lib.camera(d, 0, 1e4), 3360 * 2160),
        "cross_section": (lambda: lib.cross_section(d), 400 * 400),
    }
    result = dict(workload="golden 16-camera FTHETA rig (3360 x 2160, 90 degree fov), app defaults", gpu=gpu,
                  power_limit=limit, reps=args.reps, entry_points={})
    total = 0.0
    for name, (fn, points) in calls.items():
        ms = time_call(fn, args.reps)
        host = lib.last_host_points()
        med = float(np.median(ms))
        total += med
        result["entry_points"][name] = dict(ms=ms, ms_median=med, points=points, host_points=host,
                                            host_point_share=host / points)
    with tempfile.TemporaryDirectory() as tmp:
        flags = ["--rig=" + ru.GOLDEN_RIG, "--output_camera_id=cam0"] + [
            "--%s=%s" % (o, os.path.join(tmp, o)) for o in
            ("output_obj", "output_equirect", "output_camera", "output_cross_section")]
        t0 = time.perf_counter()
        p = ru.run_app(flags)
        wall = time.perf_counter() - t0
        assert p.returncode == 0, p.stderr[-2000:]
        result["app"] = dict(wall_s=wall, entry_points_s=total / 1e3, host_s=wall - total / 1e3,
                             ppm_bytes=sum(os.path.getsize(os.path.join(tmp, o)) for o in
                                           ("output_equirect", "output_camera", "output_cross_section")))
        if not args.no_cpu:
            ref = ru.load_ref()
            os.makedirs(os.path.join(tmp, "ref"))
            t0 = time.perf_counter()
            ref.main([f.replace(tmp, os.path.join(tmp, "ref")) for f in flags])
            result["cpu"] = dict(wall_s=time.perf_counter() - t0, threads=1, cores=os.cpu_count(),
                                 arm="the reference's main (checker build), same flags")
    line = json.dumps(result)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
