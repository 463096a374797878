"""Cost of adding particles to a running simulation (GmpmSimulator.add_particles / add_particles_sdf, csrc/emit.cuh) at the bench's scale.

Scene: the bench's two elastic spheres, 512^3 grid, 40 M particles, stepped 5 sub-steps.  Emissions: 10 k and 1 M particles into
the first sphere's model, as a host array (a lattice box above the spheres) and from a level set (a lattice-mode sphere), with fill
"all" and "empty".  Every call starts from the same state: a simulator restored from one checkpoint of the stepped scene.  Prints JSON lines: the GPU (name, power limit), then per emission the host time of the call (it
synchronises) and the per-kernel times of one call (torch.profiler's CUDA kernel records, a separate run).

    python tools/emit_bench.py [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

BITS = 9
DX = 1.0 / (1 << BITS)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def emissions():
    import numpy as np
    from claymore_b200 import samplers, sdf
    from claymore_b200._capi import SdfHeader

    def box(n_cells):   # n_cells^3 cells x 8 particles, above the spheres
        lo = np.array([200, 420, 200])
        return samplers.uniform_box(DX, tuple(lo), tuple(lo + n_cells))

    def sphere_ls(radius_cells):
        m = radius_cells + 3
        q = (np.arange(2 * m + 1) - m) * DX
        x, y, z = np.meshgrid(q, q, q, indexing="ij")
        phi = (np.sqrt(x * x + y * y + z * z) - radius_cells * DX).astype(np.float32)
        hdr = SdfHeader()
        hdr.ni = hdr.nj = hdr.nk = 2 * m + 1
        hdr.h = DX
        ls = sdf.LevelSet(hdr, np.ascontiguousarray(phi.transpose(2, 1, 0).reshape(-1)))
        return ls, (0.5 - m * DX, 0.86 - m * DX, 0.5 - m * DX), (2 * m * DX,) * 3

    out = []
    for label, cells, rad in (("10k", 11, 7), ("1M", 50, 31)):
        pos = box(cells)
        ls, off, span = sphere_ls(rad)
        for fill in ("all", "empty"):
            out.append((f"host {label} fill={fill}", lambda s, pos=pos, fill=fill: s.add_particles(0, pos, (0.0, -1.0, 0.0), fill=fill)))
            out.append((f"sdf {label} fill={fill}", lambda s, ls=ls, off=off, span=span, fill=fill:
                        s.add_particles_sdf(0, ls, off, span, (0.0, -1.0, 0.0), ppc=8, mode="lattice", fill=fill)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch
    import scenes
    from claymore_b200.simulator import GmpmSimulator

    print(json.dumps({"gpu": gpu_info()}), flush=True)
    scene = scenes.workload("spheres40m")[0]
    sim = scenes.build_engine(scene, max_blocks=scenes.max_blocks_for(scene), auto_grow=False)
    sim.step(5)
    blob = sim.save_checkpoint()
    sim.close()

    def fresh():
        s = GmpmSimulator.from_checkpoint(blob)
        s.restore(blob)
        return s

    for label, fn in emissions():
        times, added = [], 0
        for _ in range(args.reps + 1):
            s = fresh()
            s.sync()
            t0 = time.perf_counter()
            added = fn(s)
            s.sync()
            times.append((time.perf_counter() - t0) * 1e3)
            assert s.stats().error == 0
            s.close()
        s = fresh()
        s.sync()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fn(s)
            s.sync()
        s.close()
        kernels = {}
        for e in prof.key_averages():
            t = (getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)) / 1e3
            if t > 0:
                kernels[e.key[:60]] = round(t, 3)
        print(json.dumps({"emission": label, "added": added, "host_ms": [round(t, 2) for t in times[1:]],
                          "kernels_ms": dict(sorted(kernels.items(), key=lambda kv: -kv[1])[:12])}), flush=True)


if __name__ == "__main__":
    main()
