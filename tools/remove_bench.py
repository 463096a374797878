"""Cost of removing particles from a running simulation (GmpmSimulator.remove_particles / remove_rows, csrc/remove.cuh) at the
bench's scale.

Scene: the bench's two elastic spheres, 512^3 grid, 40 M particles, stepped 5 sub-steps.  Removals: about 10 k and about 1 M
particles with a box region through the top of the first sphere, and a 40 M-entry random mask (remove_rows) removing about 1 M of
model 0.  Every call starts from the same state: a simulator restored from one checkpoint of the stepped scene.  Prints JSON lines:
the GPU (name, power limit, max SM clock), then per removal the host time of the call (it synchronises), the per-kernel times of
one call (torch.profiler's CUDA kernel records, a separate run) and the select / compact pair's achieved bandwidth against the
H100 SXM's 3.35 TB/s: algorithmic bytes are the C channels of every row read once plus the survivors' rows written.

    python tools/remove_bench.py [--reps 3]
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
PEAK_BW = 3.35e12


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def removals(top, n0):
    import numpy as np
    from claymore_b200 import objects

    def slab(thickness):   # a box over the first sphere's top `thickness` (world units), every model
        return lambda s: s.remove_particles([objects.box((0.0, top - thickness, 0.0), (1.0, 1.0, 1.0))], models=[0])

    rng = np.random.default_rng(0)
    mask = rng.random(n0) < 1e6 / n0
    return [("box ~10k", slab(0.0045)), ("box ~1M", slab(0.043)), ("mask 1M of 40M rows", lambda s: s.remove_rows(0, mask))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch
    import scenes
    from claymore_b200._capi import CHANNELS
    from claymore_b200.simulator import GmpmSimulator

    print(json.dumps({"gpu": gpu_info()}), flush=True)
    scene = scenes.workload("spheres40m")[0]
    sim = scenes.build_engine(scene, max_blocks=scenes.max_blocks_for(scene), auto_grow=False)
    sim.step(5)
    blob = sim.save_checkpoint()
    top = float(sim.retrieve(0)[:, 1].max())
    n = [len(sim.retrieve(m)) for m in range(len(sim.materials))]
    chans = [CHANNELS[m] for m in sim.materials]
    sim.close()
    print(json.dumps({"rows": n}), flush=True)

    def fresh():
        s = GmpmSimulator.from_checkpoint(blob)
        s.restore(blob)
        return s

    for label, fn in removals(top, n[0]):
        times, removed = [], None
        for _ in range(args.reps + 1):
            s = fresh()
            s.sync()
            t0 = time.perf_counter()
            removed = fn(s)
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
        kernels, select_ms = {}, 0.0
        for e in prof.key_averages():
            t = (getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)) / 1e3
            if t > 0:
                kernels[e.key[:60]] = round(t, 3)
                if "Remove" in e.key:
                    select_ms += t
        # the select / compact pair of model 0: every row's C channels read once, the survivors' written once
        rows, kept = n[0], n[0] - removed[0]
        bytes_ = 4.0 * chans[0] * (rows + kept)
        print(json.dumps({"removal": label, "removed": removed, "host_ms": [round(t, 2) for t in times[1:]],
                          "select_compact_ms": round(select_ms, 3), "select_compact_TBps": round(bytes_ / (select_ms * 1e-3) / 1e12, 3) if select_ms else None,
                          "of_peak": round(bytes_ / (select_ms * 1e-3) / PEAK_BW, 3) if select_ms else None,
                          "kernels_ms": dict(sorted(kernels.items(), key=lambda kv: -kv[1])[:12])}), flush=True)


if __name__ == "__main__":
    main()
