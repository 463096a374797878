#!/usr/bin/env python
"""g2p2g time of every sub-step of a bench.py workload on one GPU, next to the sub-steps at which the scene's initial velocities
move a whole particle sub-lattice across a cell face (particles that change cell take g2p2g's slower path):
    python tools/step_profile.py [--workload spheres40m] [--steps 110]
Prints JSON lines: the GPU (name, power limit, max SM clock), the predicted crossings, one line per sub-step, and a summary.
Needs a GPU; there is no fallback."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402


def predicted_crossings(scene, dt, steps):
    """{sub-step k: particles whose cell changes in k} from the initial positions and v0 alone (no forces): a particle changes
    cell in sub-step k when round((p + k v dt) / dx) != round((p + (k - 1) v dt) / dx) along some axis.  Counted per axis on
    the distinct coordinates, so a particle crossing along two axes in one sub-step counts twice."""
    dx = 1.0 / (1 << scene["domain_bits"])
    k = np.arange(steps + 1, dtype=np.float64)
    out = {}
    for m in scene["models"]:
        for d in range(3):
            v = float(m["v0"][d])
            if v == 0.0:
                continue
            coord, count = np.unique(m["pos"][:, d], return_counts=True)
            cell = np.rint((coord[:, None].astype(np.float64) + k[None, :] * v * dt) / dx)
            moved = cell[:, 1:] != cell[:, :-1]          # [coordinate, sub-step 1..steps]
            for s in np.nonzero(moved.any(0))[0]:
                out[int(s) + 1] = out.get(int(s) + 1, 0) + int(count[moved[:, s]].sum())
    return dict(sorted(out.items()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="spheres40m")
    ap.add_argument("--steps", type=int, default=110)
    ap.add_argument("--dt", type=float, default=1e-4)
    ap.add_argument("--max-ppc", type=int, default=128)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("step_profile.py needs a CUDA device")
    from claymore_b200 import scenes

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], stdout=subprocess.PIPE, text=True, check=True)
    print(json.dumps({"gpu": smi.stdout.strip().splitlines()[1:]}))

    scene = scenes.workload(args.workload)[0]
    n = scenes.n_particles(scene)
    cross = predicted_crossings(scene, args.dt, args.steps)
    bursts = [k for k, c in cross.items() if c >= 0.01 * n]   # sub-steps where at least 1 % of the particles change cell
    print(json.dumps({"workload": args.workload, "particles": n, "predicted_crossings": cross, "burst_substeps": bursts}))

    stream = torch.cuda.Stream()
    sim = scenes.build_engine(scene, dt=args.dt, max_blocks=scenes.max_blocks_for(scene), max_ppc=args.max_ppc, stream=stream.cuda_stream, auto_grow=False)
    sim.profile(True)
    ms = []
    for k in range(1, args.steps + 1):
        sim.step(1)
        t, launches = sim.profile_read()
        ms.append(t)
        print(json.dumps({"substep": k, "g2p2g_ms": round(t, 4), "launches": launches}))
    sim.profile(False)
    st = sim.stats()
    sim.close()
    assert st.error == 0, f"engine error bits {st.error}"

    # burst sub-steps against the median of the others (the first few sub-steps warm up caches and modules)
    calm = [t for k, t in enumerate(ms, 1) if k not in bursts and k > 3]
    med = statistics.median(calm)
    print(json.dumps({"summary": True, "median_other_ms": round(med, 4),
                      "burst_ms": {k: round(ms[k - 1], 4) for k in bursts if k <= args.steps},
                      "burst_over_median": {k: round(ms[k - 1] / med - 1.0, 4) for k in bursts if k <= args.steps},
                      "mean_ms": round(sum(ms[3:]) / len(ms[3:]), 4)}))


if __name__ == "__main__":
    main()
