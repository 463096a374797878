#!/usr/bin/env python
"""Time and memory traffic of every kernel of a sub-step on a bench.py workload, one GPU:
    python tools/tail_profile.py [--workload spheres40m] [--steps 100] [--warmup 5]
After the warm-up, `steps` sub-steps run as plain stream launches under torch.profiler (CUDA activities), which gives the time of
each kernel by name; the same sub-steps carry the driver's phase events (profile_phases) as a cross-check.  Beside each kernel's
time stand the bytes its algorithm has to move, from the block counts, particle count, model count and max_ppc of stats(), the
rate that makes, and that rate's share of the H100 SXM's 3.35 TB/s of HBM3 (data sheet, 700 W card).  g2p2g is listed by time only:
bench.py holds its byte model.
Prints JSON lines: the GPU (name, power limit, max SM clock), the byte model, one line per kernel, the phases.
Needs a GPU; without one it prints the byte model for block counts estimated from the scene's start positions and fails."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
GRID_BLOCK = 1024      # 4 channels x 64 cells x 4 bytes
COUNT_ROW = 256        # 64 cell counts
OFFS_ROW = 128         # 64 cell offsets (u16)
SECTOR = 32


def byte_model(pbc, nbc, ebc, particles, models, max_ppc):
    """{kernel: bytes one sub-step's launch has to move}.  pbc / nbc / ebc: particle, + neighbour, + exterior blocks."""
    tags_in = particles * 4   # the eight or so tags of a cell are its first slot group: 32 contiguous bytes of the block's 2 KiB group 0
    return {
        # read + write every grid block, zero the next grid's, zero every model's cell counts over the exterior blocks
        "grid_update_kernel": nbc * 3 * GRID_BLOCK + ebc * models * COUNT_ROW,
        # every cell-count row once, a total per block and model out, the stale table entries and keys
        "summary_kernel": ebc * models * (COUNT_ROW + 4) + ebc * (12 + 4),
        # totals in; per particle block: keys in and out, a table entry, and per model holding particles there (about one per
        # block) the count row, the cell offsets, size and bin offset; every tag in and out
        "rebuild_kernel": ebc * models * 4 + pbc * (24 + 4) + pbc * (COUNT_ROW + OFFS_ROW + 8) + tags_in + particles * 4,
        # 8 / 27 probes per particle block: a key read, a table entry read (a CAS when new), a key written per new block
        "register_blocks_kernel(neighbour)": pbc * (12 + 8 * 4) + (nbc - pbc) * (12 + 4),
        "register_blocks_kernel(exterior)": pbc * (12 + 27 * 4) + (ebc - nbc) * (12 + 4),
        # every block of the new numbering: key, old table entry, 1 KiB in, 1 KiB out
        "carry_grid_kernel": nbc * (12 + 4 + 2 * GRID_BLOCK),
    }


def estimated_counts(scene):
    """block counts of the scene's start positions (no device): blocks holding particles, + the 2^3 neighbours, + the 3^3 exterior"""
    bits = scene["domain_bits"]
    key = lambda b: (b[:, 0].astype(np.int64) << 40) | (b[:, 1].astype(np.int64) << 20) | b[:, 2].astype(np.int64)  # noqa: E731
    blocks = np.concatenate([np.unique(((np.rint(m["pos"] * (1 << bits)).astype(np.int64) - 2) >> 2), axis=0) for m in scene["models"]])
    blocks = np.unique(blocks, axis=0)
    def dilate(lo, hi):
        offs = np.array([(i, j, k) for i in range(lo, hi) for j in range(lo, hi) for k in range(lo, hi)], np.int64)
        return len(np.unique(key((blocks[:, None, :] + offs[None, :, :]).reshape(-1, 3))))
    return len(blocks), dilate(0, 2), dilate(-1, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="spheres40m")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--dt", type=float, default=1e-4)
    ap.add_argument("--max-ppc", type=int, default=0)
    ap.add_argument("--scene", default=None, help="a function of claymore_b200.scenes in place of a workload (small scenes)")
    args = ap.parse_args()

    import torch
    from claymore_b200 import scenes
    scene = getattr(scenes, args.scene)() if args.scene else scenes.workload(args.workload)[0]
    label = args.scene or args.workload
    max_ppc = args.max_ppc or (32 if label.startswith("mixed") else 128)   # bench.py's rule
    n, nm = scenes.n_particles(scene), len(scene["models"])
    if not torch.cuda.is_available():
        pbc, nbc, ebc = estimated_counts(scene)
        print(json.dumps({"workload": label, "particles": n, "models": nm, "max_ppc": max_ppc, "blocks_estimated": [pbc, nbc, ebc],
                          "bytes": byte_model(pbc, nbc, ebc, n, nm, max_ppc)}))
        raise SystemExit("tail_profile.py needs a CUDA device: nothing was timed")
    from torch.profiler import ProfilerActivity, profile

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], stdout=subprocess.PIPE, text=True, check=True)
    print(json.dumps({"gpu": smi.stdout.strip().splitlines()[1:]}))

    stream = torch.cuda.Stream()
    sim = scenes.build_engine(scene, dt=args.dt, max_blocks=scenes.max_blocks_for(scene), max_ppc=max_ppc, stream=stream.cuda_stream, auto_grow=False)
    sim.step(args.warmup)
    sim.sync()
    sim.profile(True)   # plain stream launches (a replayed graph would hide nothing, but the phase events need them)
    sim.step(2)
    sim.sync()
    sim.profile_phases(), sim.profile_read()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        sim.step(args.steps)
        sim.sync()
    phases = {k: round(v / args.steps, 4) for k, v in sim.profile_phases().items()}
    sim.profile_read()
    sim.profile(False)
    st = sim.stats()
    sim.close()
    assert st.error == 0, f"engine error bits {st.error}"

    pbc, nbc, ebc = st.particle_block_count, st.neighbor_block_count, st.exterior_block_count
    model = byte_model(pbc, nbc, ebc, n, nm, max_ppc)
    print(json.dumps({"workload": label, "particles": n, "models": nm, "max_ppc": max_ppc, "blocks": [pbc, nbc, ebc], "steps": args.steps, "bytes": model}))

    # the two registration launches of a sub-step share a kernel: told apart by their order on the stream (neighbour first)
    rows, reg = {}, []
    for e in prof.events():
        name = e.name.split("(")[0].split("<")[0].split("::")[-1]
        if not name.endswith("_kernel"):
            continue
        if name == "register_blocks_kernel":
            reg.append(e)
            continue
        r = rows.setdefault(name, [0.0, 0])
        r[0] += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        r[1] += 1
    reg.sort(key=lambda e: e.time_range.start)
    for i, e in enumerate(reg):
        r = rows.setdefault("register_blocks_kernel(%s)" % ("neighbour" if i % 2 == 0 else "exterior"), [0.0, 0])
        r[0] += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        r[1] += 1
    total = 0.0
    for name, (us, count) in sorted(rows.items(), key=lambda kv: -kv[1][0]):
        ms = us / 1e3 / args.steps
        total += ms
        line = {"kernel": name, "launches_per_step": round(count / args.steps, 2), "ms_per_step": round(ms, 4)}
        if name in model:
            rate = model[name] / (ms * 1e-3)
            line.update(bytes=model[name], gb_per_s=round(rate / 1e9, 1), share_of_3350_gb_per_s=round(rate / HBM_BYTES_PER_S, 3),
                        ms_at_3350_gb_per_s=round(model[name] / HBM_BYTES_PER_S * 1e3, 4))
        print(json.dumps(line))
    print(json.dumps({"kernels_ms_per_step": round(total, 4), "phases_ms_per_step": phases, "phases_sum": round(sum(phases.values()), 4)}))


if __name__ == "__main__":
    main()
