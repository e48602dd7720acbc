#!/usr/bin/env python3
"""Kernel-by-kernel time of the filtered sweep on one headline destination: 16-camera FTHETA ring, 2048 x 2048,
128 candidates from 0.5 m to 10^4 m (the scene and rig of bench.py's bf128_l0).

The whole derp_brute_force call is timed with CUDA events; the four kernels of the filtered sweep (sweepLowerKernel,
sweepSeedKernel, refineListKernel, refineKernel) are timed from the CUDA activity trace of torch.profiler, in a separate
pass so that tracing does not disturb the event timing.  The GPU's name and power limit are read in the same run.

Prints one JSON line.  Writes nothing in the tree unless --out is given.  DERP_B200_LIB selects another build of the
library, so that builds can be compared in one session by alternating runs of this script."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from facebook360_dep_b200 import capi, synth  # noqa: E402

KERNELS = ("sweepLowerKernel", "sweepSeedKernel", "refineListKernel", "refineKernel")


def gpu_conditions():
    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        out["power_limit_w"] = float(q.stdout.strip().splitlines()[0])
    except Exception as e:  # nvidia-smi missing or unreadable
        out["power_limit_w"] = "unknown (%s)" % type(e).__name__
    return out


def kernel_times(fn, reps):
    """Mean device time per call of fn, in ms, of every kernel named in KERNELS (from the CUDA activity trace)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        events = json.load(open(path)).get("traceEvents", [])
    us = {k: 0.0 for k in KERNELS}
    for e in events:
        if e.get("cat") != "kernel":
            continue
        name = e.get("name", "")
        for k in KERNELS:
            if k + "<" in name or k + "(" in name:
                us[k] += float(e.get("dur", 0.0))
    return {k: v / 1e3 / reps for k, v in us.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dst", type=int, default=0)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--label", default=None, help="a name for this build in the output line")
    ap.add_argument("--out", default=None, help="also append the JSON line to this file")
    a = ap.parse_args()
    S, W, H, D = 16, 2048, 2048, 128
    rig = synth.ring_rig(S, W, H, kind="FTHETA")
    colors, _ = synth.render_rig(rig, W, H, scene=synth.Scene(seed=42), device="cuda")
    torch.cuda.empty_cache()
    lib = capi.load_cuda()
    ctx = capi.Context(lib, capi.rig_descs(rig))
    stream = torch.cuda.current_stream()
    ctx.set_stream(stream.cuda_stream)
    ctx.level_begin(W, H)
    ctx.set_colors(colors)
    ctx.set_sweep_mode(2)  # filtered
    ctx.reproject(a.dst)

    def step():
        ctx.brute_force(a.dst, num_depths=D, min_depth_m=0.5, max_depth_m=1e4, want_index=False)

    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(a.reps):
        step()
    e1.record(stream)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.reps
    evals, hits = ctx.get_counters()
    refined, seeds = ctx.sweep_stats()
    per_kernel = kernel_times(step, a.reps)
    ctx.close()
    result = {"tool": "tools/bound_pass_bench.py", "label": a.label, "library": os.path.relpath(capi.CUDA_LIB),
              "gpu": gpu_conditions(),
              "config": {"cameras": S, "camera_model": "FTHETA ring", "width": W, "height": H, "candidates": D,
                         "depth_range_m": [0.5, 1e4], "destination": a.dst, "reps": a.reps, "warmup": a.warmup},
              "ms_per_destination": ms, "kernel_ms": per_kernel,
              "cost_evaluations": evals, "source_hits": hits,
              "exact_evaluations_fraction": (refined + seeds) / max(1, evals)}
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
