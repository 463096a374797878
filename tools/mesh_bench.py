"""Times mesh level sets (claymore_b200.mesh) on one GPU: the torus of tests/golden at lattices of about 100^3, 200^3 and 400^3
nodes and a floor-plus-torus mesh.  Per case: the whole host call (median of --reps, after one warm-up), the kernel time of each
stage from torch.profiler (setup + scan, band, crossings, sweeps, sign), the sweeps' dependent plane steps 16 (ni + nj + nk - 5),
and SDFGen's host time for the same lattice (oracle/_ref/libclaymore_ref_sdfgen.so, one thread) where it is built and the lattice
is at most --sdfgen-max nodes.  Prints one JSON line per case, with the GPU's name and power limit.

    python tools/mesh_bench.py [--reps 5] [--sdfgen-max 3e6]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import mesh_cases as M  # noqa: E402
from claymore_b200 import mesh  # noqa: E402

STAGES = {"mesh_setup_kernel": "setup", "mesh_scan": "setup", "mesh_init_kernel": "setup", "mesh_band_kernel": "band",
          "mesh_cross_kernel": "crossings", "mesh_sweep_kernel": "sweeps", "mesh_sign_kernel": "sign"}


def cases():
    v, t = M.torus()
    floor_v = np.asarray([[-3, -0.5, -3], [3, -0.5, -3], [3, -0.5, 3], [-3, -0.5, 3]], np.float32)
    fv = np.vstack([v, floor_v]).astype(np.float32)
    ft = np.vstack([t, np.asarray([[0, 1, 2], [0, 2, 3]]) + len(v)]).astype(np.int32)
    return {"torus_100": (v, t, 0.02), "torus_200": (v, t, 0.01), "torus_400": (v, t, 0.005), "floor_torus": (fv, ft, 0.02)}


def stage_times(m, h):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        mesh.levelset(m, h)
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        for k, s in STAGES.items():
            if k in e.name and e.device_type.name == "CUDA":
                out[s] = out.get(s, 0.0) + e.device_time / 1e3
    return {k: round(v, 3) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sdfgen-max", type=float, default=3e6)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    L = M.shim()
    for name, (v, t, h) in cases().items():
        m = mesh.Mesh(v, t)
        hdr = mesh.header(m, h)
        n = (hdr.ni, hdr.nj, hdr.nk)
        mesh.levelset(m, h)
        ts = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            ls = mesh.levelset(m, h)
            ts.append(time.perf_counter() - t0)
        r = {"case": name, "triangles": len(t), "nodes": list(n), "plane_steps": 16 * (sum(n) - 5), "call_ms": round(1e3 * float(np.median(ts)), 2),
             "stage_ms": stage_times(m, h), "gpu": gpu}
        if L is not None and np.prod(n) <= a.sdfgen_max:
            t0 = time.perf_counter()
            _, _, ref = M.ref_level_set(L, v, t, h, 1, 1)
            r["sdfgen_ms"] = round(1e3 * (time.perf_counter() - t0), 1)
            r["bitwise_equal_sdfgen"] = bool(np.array_equal(ref.view(np.uint32), ls.phi.view(np.uint32)))
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
