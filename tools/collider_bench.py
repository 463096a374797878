"""Cost of the signed-distance collider on the bench's flagship workload.

Runs the 40 M-particle two-sphere scene (bench.py's default, 512^3 grid) with a static sticky floor box under the spheres and
with no collider, alternating the two in one process, and prints JSON lines: the GPU (name, power limit, max SM clock), then per
run the sub-step time (CUDA events, graph replay) and the per-phase milliseconds of profile_phases (grid_update first).

    python tools/collider_bench.py [--steps 50] [--warmup 10] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def run(scene, field, args, stream):
    import torch
    from claymore_b200 import scenes
    sim = scenes.build_engine(scene, dt=args.dt, max_blocks=scenes.max_blocks_for(scene), stream=stream.cuda_stream, auto_grow=False)
    if field is not None:
        sim.set_collider(field[0], field[1], type="sticky")
    sim.step(args.warmup)
    sim.sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    sim.step(args.steps)
    e1.record(stream)
    torch.cuda.synchronize()
    substep_ms = e0.elapsed_time(e1) / args.steps
    sim.profile(True)
    sim.step(args.steps)
    phases = {k: round(v / args.steps, 4) for k, v in sim.profile_phases().items()}
    sim.profile_read()
    sim.profile(False)
    st = sim.stats()
    sim.close()
    assert st.error == 0, f"engine error bits {st.error}"
    return {"substep_ms": round(substep_ms, 4), "phases_ms": phases}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--dt", type=float, default=1e-4)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("collider_bench.py needs a CUDA device")
    from claymore_b200 import levelset, scenes
    from claymore_b200._capi import Config

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], stdout=subprocess.PIPE, text=True, check=True)
    print(json.dumps({"gpu": smi.stdout.strip().splitlines()[1:]}), flush=True)
    scene = scenes.workload("spheres40m")[0]
    # the spheres' lowest point is y = 0.5 - 0.1645: the floor's top sits half a cell under it
    top = 0.5 - 0.1645 - 0.5 / (1 << scene["domain_bits"])
    field = levelset.box(Config(domain_bits=scene["domain_bits"]), (0.1, 0.1, 0.1), (0.9, top, 0.9))
    stream = torch.cuda.Stream()
    for r in range(args.rounds):
        order = ("floor", "none") if r % 2 == 0 else ("none", "floor")
        for name in order:
            res = run(scene, field if name == "floor" else None, args, stream)
            print(json.dumps({"round": r, "collider": name, "steps": args.steps, **res}), flush=True)


if __name__ == "__main__":
    main()
