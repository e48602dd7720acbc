"""Times RigSimulator's renders (include/derp_rigsim.h) on one GPU and writes one JSON file per workload.

  ftheta_ring15 : the reference app's defaults: --scene icosahedron (250 icosahedrons), --mode ftheta_ring with 14
                  FTHETA cameras of 300 x 400 on a 0.218 m ring plus the top camera, --anti_alias_supersample 1
  ring16_2048   : a 16-camera FTHETA ring of 2048 x 2048 at --anti_alias_supersample 2 (the depth benchmark's rig size)
  mono_eqr      : --mode mono_eqr at the default 3080 x 1540 and --anti_alias_supersample 2
Each library call is timed with CUDA events after a warm-up call (outputs in device memory for the cameras, host
arrays for the equirect, whose copy back is inside the window), with the share of rays whose sky texel the host
resolved.  The CPU arm runs the checker (the reference's own renderCamera, oracle/rigsim.mk) on the first workload,
one camera per host thread as the reference app does.
Usage: python tools/rig_simulator_bench.py [--outdir profiles] [--reps 5] [--no-cpu]"""
import argparse
import json
import math
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from facebook360_dep_b200 import capi  # noqa: E402
from tests import rigsim_util as ru  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "not measured"


def ftheta_ring15():
    """The app's default --mode ftheta_ring rig (14 ring cameras plus the top camera), as its --rig_out writes it."""
    with tempfile.TemporaryDirectory() as tmp:
        sky, rig = os.path.join(tmp, "sky.png"), os.path.join(tmp, "rig.json")
        ru.write_skybox(sky, ru.skybox(8, 4))
        subprocess.run([os.path.join(ROOT, "facebook360_dep_b200", "bin", "RigSimulator"), "--mode=ftheta_ring",
                        "--skybox_path=" + sky, "--rig_out=" + rig], check=True, capture_output=True)
        with open(rig) as f:
            return capi.rig_descs(json.load(f))


def time_call(fn, reps):
    fn()  # warm-up: module load, scratch allocation
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(reps):
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--outdir", default=os.path.join(ROOT, "profiles"))
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-cpu", action="store_true")
    args = ap.parse_args()
    gpu, limit = gpu_info()
    sim = capi.RigSim(capi.load_cuda())
    sim.srand(1)
    scene = sim.scene("icosahedron")
    sky = ru.skybox(2048, 1024, seed=0)
    results = []

    def cameras(name, descs, aas):
        outs = [[torch.empty((int(d.resolution[1]), int(d.resolution[0]), 3), device="cuda") for d in descs],
                [torch.empty((int(d.resolution[1]), int(d.resolution[0])), device="cuda") for d in descs]]
        ptrs = ([t.data_ptr() for t in outs[0]], [t.data_ptr() for t in outs[1]])
        ms = time_call(lambda: sim.render_cameras(scene, descs, sky, outs=ptrs, aas=aas), args.reps)
        host, rays = sim.last_host_rays()
        return dict(workload=name, cameras=len(descs), width=int(descs[0].resolution[0]),
                    height=int(descs[0].resolution[1]), aas=aas, rays=rays, host_rays=host,
                    host_ray_share=host / rays, ms=ms, ms_median=float(np.median(ms)),
                    grays_per_s=rays / (float(np.median(ms)) * 1e-3) / 1e9)

    r = cameras("ftheta_ring15", ftheta_ring15(), 1)
    if not args.no_cpu:
        ref = ru.load_ref()
        if ref is None:
            raise SystemExit("the CPU arm needs the checker (oracle/rigsim.mk)")
        ref.build("icosahedron", seed=1)
        ref.set_render(sky)
        descs = ftheta_ring15()
        t0 = time.perf_counter()
        with ThreadPoolExecutor(len(descs)) as ex:
            list(ex.map(ref.render_camera, descs))
        r["cpu_ms"] = (time.perf_counter() - t0) * 1e3
        r["cpu_threads"] = len(descs)
        r["cpu_cores"] = os.cpu_count()
        r["cpu_arm"] = "the reference's renderCamera (checker build), one camera per thread"
    results.append(r)
    results.append(cameras("ring16_2048", ru.ring_descs(16, 2048, 2048), 2))
    ms = time_call(lambda: sim.render_equirect(scene, 3080, 1540, sky, aas=2), args.reps)
    host, rays = sim.last_host_rays()
    results.append(dict(workload="mono_eqr", width=3080, height=1540, aas=2, rays=rays, host_rays=host,
                        host_ray_share=host / rays, ms=ms, ms_median=float(np.median(ms)),
                        grays_per_s=rays / (float(np.median(ms)) * 1e-3) / 1e9,
                        note="host outputs: the copy back is inside the timed window"))
    os.makedirs(args.outdir, exist_ok=True)
    for r in results:
        r.update(gpu=gpu, power_limit=limit, scene="icosahedron, 250 icosahedrons, srand(1)",
                 skybox="2048 x 1024 seeded noise")
        line = json.dumps(r)
        print(line)
        with open(os.path.join(args.outdir, "h100_rigsim_%s.json" % r["workload"]), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
