#!/usr/bin/env python3
"""Level-0 brute force on a rig of more than 32 cameras (the 64-bit visibility-mask kernels): 48-camera FTHETA ring,
1024 x 1024, 128 candidates, one destination per step, in the plain and the filtered sweep mode.

Prints one JSON line: throughput in Mpix·cand/s (cost evaluations per second), v̄ = source hits / cost evaluations, the
launched CTA shape of the sweep kernels (read from the CUDA activity trace of torch.profiler), and the GPU's name and
power limit read in the same run.  Writes nothing in the tree unless --out is given."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from facebook360_dep_b200 import capi, synth  # noqa: E402


def gpu_conditions():
    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        out["power_limit_w"] = float(q.stdout.strip().splitlines()[0])
    except Exception as e:  # nvidia-smi missing or unreadable
        out["power_limit_w"] = "unknown (%s)" % type(e).__name__
    return out


def launch_shapes(fn):
    """grid / block / dynamic shared memory / registers of the sweep kernels one call of fn launches."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        events = json.load(open(path)).get("traceEvents", [])
    shapes = {}
    for e in events:
        name = e.get("name", "")
        if e.get("cat") == "kernel" and ("sweepKernel" in name or "sweepLowerKernel" in name):
            a = e.get("args", {})
            key = name.split("(")[0].replace("void ", "")
            shapes[key] = {"grid": a.get("grid"), "block": a.get("block"), "dynamic_smem_bytes": a.get("shared memory"),
                           "registers_per_thread": a.get("registers per thread")}
    return shapes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cams", type=int, default=48)
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--candidates", type=int, default=128)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    W = H = a.size
    rig = synth.ring_rig(a.cams, W, H, kind="FTHETA")
    colors, _ = synth.render_rig(rig, W, H, device="cuda")
    torch.cuda.empty_cache()
    ctx = capi.Context(capi.load_cuda(), capi.rig_descs(rig))
    stream = torch.cuda.current_stream()
    ctx.set_stream(stream.cuda_stream)
    ctx.level_begin(W, H)
    ctx.set_colors(colors)
    dsts = [(i * 7) % a.cams for i in range(a.steps)]
    result = {"tool": "tools/wide_rig_bench.py", "gpu": gpu_conditions(),
              "config": {"cameras": a.cams, "camera_model": "FTHETA ring", "width": W, "height": H, "candidates": a.candidates,
                         "level": 0, "destinations_timed": dsts, "steps": a.steps, "warmup": a.warmup,
                         "timed": "derp_brute_force of one destination per step (after its derp_reproject), CUDA events"},
              "modes": {}}
    for mode, label in ((1, "plain"), (2, "filtered")):
        ctx.set_sweep_mode(mode)

        def step(d):
            ctx.brute_force(d, num_depths=a.candidates, want_index=False)

        for i in range(a.warmup):
            ctx.reproject(dsts[i % len(dsts)])
            step(dsts[i % len(dsts)])
        torch.cuda.synchronize()
        ms, evals, hits = 0.0, 0, 0
        for d in dsts:
            ctx.reproject(d)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            step(d)
            e1.record(stream)
            torch.cuda.synchronize()
            ms += e0.elapsed_time(e1)
            ev, h = ctx.get_counters()
            evals += ev
            hits += h
        result["modes"][label] = {"value": evals / (ms / 1e3) / 1e6, "unit": "Mpix·cand/s", "ms_per_step": ms / len(dsts),
                                  "v_bar": hits / evals, "cost_evaluations_per_step": evals // len(dsts),
                                  "launches": launch_shapes(lambda: step(dsts[-1]))}
    ctx.close()
    line = json.dumps(result, ensure_ascii=False)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
