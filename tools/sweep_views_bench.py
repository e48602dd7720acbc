"""Times the sweep-view slices on one GPU and prints one JSON line.

  overlaps : derp_sweep_overlaps for one destination of the default GenerateCameraOverlaps shape (the 16-camera FTHETA
             ring of synth.py at 3360 x 2160, --scale 0.5, 50 slices), images and output resident on the device, CUDA
             events around the call; reported per (destination, slice).
  equirect : derp_sweep_equirect of a 512-row equirect at 50 depths, reported per depth.
  vbar     : contributing (sample, camera) pairs per sample (derp_sweep_last_hits).
  app      : GenerateCameraOverlaps on a synthetic dataset of the same shape for one destination (--cameras=cam0),
             wall time split into decode / device / encode as the app logs it.
  reference: the reference's own projectSrcsToDst (oracle/_ref checker) on one host thread for a few slices,
             extrapolated to 16 destinations x 50 slices (labelled as such; not measured at that size).
Usage: python tools/sweep_views_bench.py [--skip-app] [--ref-slices 2]"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from facebook360_dep_b200 import capi, synth  # noqa: E402
from tests import sweep_oracle, sweep_util as su  # noqa: E402


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return out
    except Exception:
        return "not measured"


def timed(fn, reps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-app", action="store_true")
    ap.add_argument("--ref-slices", type=int, default=2)
    a = ap.parse_args()
    lib = capi.SweepView(capi.load_cuda())
    rig = synth.ring_rig(16, 3360, 2160, kind="FTHETA")
    descs = capi.rescaled_descs(capi.rig_descs(rig), 0.5)
    rng = np.random.default_rng(0)
    host = [rng.random((1080, 1680, 4), dtype=np.float32) for _ in range(16)]
    dev = [torch.from_numpy(x).cuda() for x in host]
    ptrs = (capi.C.c_void_p * 16)(*[t.data_ptr() for t in dev])
    sizes = np.array([[1680, 1080]] * 16, np.int32).reshape(-1)
    disp = su.slice_disparities(50, 1, 10)
    d_disp = np.ascontiguousarray(disp)
    out = torch.empty((50, 1080, 1680, 4), dtype=torch.float32, device="cuda")

    def run_overlaps():
        rc = lib.lib.derp_sweep_overlaps(0, descs, 16, ptrs, sizes.ctypes.data, 0, d_disp.ctypes.data, 50, out.data_ptr())
        assert rc == 0, lib.lib.derp_last_error()
    ms = timed(run_overlaps, 3)
    hits = lib.last_hits()
    samples = 50 * 1080 * 1680
    eq_depths = su.equirect_depths(50, 1.0, 10.0)
    eq_out = [torch.empty((512, 1024, 4), dtype=torch.float32, device="cuda") for _ in range(50)]
    eq_ptrs = (capi.C.c_void_p * 50)(*[t.data_ptr() for t in eq_out])

    def run_equirect():
        rc = lib.lib.derp_sweep_equirect(0, descs, 16, -1, ptrs, sizes.ctypes.data, 512, eq_depths.ctypes.data, 50, None,
                                         0, eq_ptrs)
        assert rc == 0, lib.lib.derp_last_error()
    eq_ms = timed(run_equirect, 3)
    eq_hits = lib.last_hits()
    result = {
        "metric": "GenerateCameraOverlaps / GenerateEquirect slices, 16-cam FTHETA ring 3360x2160 at --scale 0.5",
        "gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(),
        "overlaps_ms_per_dst_slice": ms / 50, "overlaps_ms_per_dst_50_slices": ms,
        "overlaps_vbar": hits / samples,
        "equirect_512_ms_per_depth": eq_ms / 50, "equirect_vbar": eq_hits / (50 * 512 * 1024),
    }
    ref = sweep_oracle.load_overlaps_ref()
    if ref is not None and a.ref_slices > 0:
        t = time.perf_counter()
        ref.overlaps(descs, host, 0, disp[:a.ref_slices])
        per = (time.perf_counter() - t) / a.ref_slices
        result["reference_one_thread_s_per_dst_slice"] = per
        result["reference_one_thread_s_16dst_50slices_extrapolated"] = per * 16 * 50
    else:
        result["reference_one_thread_s_per_dst_slice"] = "not measured"
    if not a.skip_app:
        with tempfile.TemporaryDirectory() as tmp:
            rng = np.random.default_rng(1)
            json.dump(rig, open(os.path.join(tmp, "rig.json"), "w"))
            for c in rig["cameras"]:
                os.makedirs(os.path.join(tmp, "color", c["id"]))
                su.write_png(os.path.join(tmp, "color", c["id"], "000000.png"),
                             rng.integers(0, 256, (2160, 3360, 4), np.uint8))
            app = os.path.join(ROOT, "facebook360_dep_b200", "bin", "GenerateCameraOverlaps")
            t = time.perf_counter()
            p = subprocess.run([app, "--rig=" + os.path.join(tmp, "rig.json"), "--color=" + os.path.join(tmp, "color"),
                                "--output=" + os.path.join(tmp, "out"), "--cameras=cam0"], capture_output=True,
                               text=True)
            wall = time.perf_counter() - t
            assert p.returncode == 0, p.stderr[-2000:]
            m = re.search(r"Timing: decode ([\d.e+]+) ms, device ([\d.e+]+) ms, encode ([\d.e+]+) ms", p.stderr)
            result["app_one_dst_50_slices"] = {"wall_s": wall, "decode_ms": float(m.group(1)),
                                               "device_incl_copy_back_ms": float(m.group(2)),
                                               "encode_ms_summed_over_threads": float(m.group(3))}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
