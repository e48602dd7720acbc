#!/usr/bin/env python3
"""Stage times of CreateObjFromDisparityEquirect at SimpleMeshRenderer's default equirect size (3072 x 1536: 4.7 M vertexes,
up to 9.4 M faces): PNG load (io::loadFloat through IoSelfTest), resize + mesh on the GPU (CUDA events around
derp_equirect_mesh with device-resident input and output), the whole app without simplification (load, mesh, OBJ
write), the reference's mesh functions from oracle/_ref on the host; and the sequential simplifier to 200 k faces, the
library's and the reference's, at a quarter of the size (1536 x 768), where the reference's still finishes in minutes.
Prints one JSON line; --out also writes it to a file.  Usage: python tools/eqr_obj_bench.py [--out FILE] [--reps N]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import cv2
    import torch
    from facebook360_dep_b200 import capi
    from tests import eqrmesh_oracle
    from tests.test_eqr_obj import APP, jumps

    cuda = capi.EqrMesh(capi.load_cuda())
    W, H = 3072, 1536
    d = jumps(W, H, 3)
    res = {"gpu": torch.cuda.get_device_name(0), "size": [W, H]}
    res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                        capture_output=True, text=True).stdout.strip()
    with tempfile.TemporaryDirectory() as tmp:
        png = os.path.join(tmp, "disp.png")
        cv2.imwrite(png, np.clip(d * 65535.0, 0, 65535).astype(np.uint16))
        t0 = time.perf_counter()
        subprocess.run([os.path.join(ROOT, "facebook360_dep_b200", "bin", "IoSelfTest"), "--mode=float", "--in=" + png,
                        "--out=" + os.path.join(tmp, "d.bin")], check=True)
        res["load_s"] = time.perf_counter() - t0
        dev = torch.from_numpy(d).cuda()
        cells = W * H
        vtx = torch.empty(cells * 3, dtype=torch.float64, device="cuda")
        idx = torch.empty(cells * 6, dtype=torch.int32, device="cuda")
        nv, nf = capi.C.c_uint64(), capi.C.c_uint64()
        for scale in (1.0, 0.5):
            times = []
            for r in range(args.reps + 1):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                cuda._check(cuda.lib.derp_equirect_mesh(0, dev.data_ptr(), W, H, scale, 700.0, 0.95, vtx.data_ptr(),
                                                       idx.data_ptr(), capi.C.byref(nv), capi.C.byref(nf)))
                b.record()
                torch.cuda.synchronize()
                if r:
                    times.append(a.elapsed_time(b))
            res["gpu_mesh_ms_scale_%g" % scale] = {"min": min(times), "median": float(np.median(times))}
        res["faces"] = nf.value
        print(json.dumps(res), flush=True)
        t0 = time.perf_counter()
        subprocess.run([APP, "--input_png_disp=" + png, "--input_png_color=c.png", "--output_obj=" + os.path.join(tmp, "m.obj"),
                        "--strictness=0"], check=True, capture_output=True)
        res["app_unsimplified_s"] = time.perf_counter() - t0
        print(json.dumps(res), flush=True)
        ref = eqrmesh_oracle.load_ref()
        quarter = jumps(W // 2, H // 2, 3)
        for name, lib in (("", cuda), ("ref_", ref)):
            if lib is None:
                continue
            if name:
                t0 = time.perf_counter()
                lib.mesh(d)
                res["ref_mesh_s"] = time.perf_counter() - t0
            t0 = time.perf_counter()
            lib.mesh(quarter, num_faces=200000, strictness=0.8)
            res[name + "mesh_and_simplify_200k_s_1536x768"] = time.perf_counter() - t0
            print(json.dumps(res), flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
