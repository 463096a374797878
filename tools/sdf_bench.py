"""Cost of sampling particle models from level sets (claymore_b200.sdf, csrc/sdf.cuh) at the bench's scale.

Workloads, 512^3 grid:
  * lattice: the bench scene's two spheres (radius 0.1645 at x = 0.3 / 0.7) as level sets whose nodes are the simulation nodes,
    ppc 8: 40 M particles, the flagship scene's count;
  * random:  one sphere level set (radius 0.207, h = dx) sampled at ppc 8: 40 M particles expected.
Prints JSON lines: the GPU (name, power limit, SM clock), then per workload the classify / count / write kernel times
(torch.profiler's CUPTI kernel records, summed over the launches of one sampling, averaged over --reps after a warm-up), the
algorithmic bytes (4 B per level-set node read, 12 B per particle written) and their share of the 3.35 TB/s data-sheet bandwidth,
and the host time of init_model_sdf against samplers.sphere + init_model for the lattice spheres, in the same run.

    python tools/sdf_bench.py [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

PEAK_BW = 3.35e12  # H100 SXM HBM3 data sheet
BITS = 9
DX = 1.0 / (1 << BITS)


def sphere_level_set(center, radius):
    import numpy as np
    import sdf_ref as R
    from claymore_b200 import sdf
    from claymore_b200._capi import SdfHeader
    m = int(np.ceil((radius + 3 * DX) / DX))
    n = (2 * m + 1,) * 3
    origin = np.asarray(center) - m * DX
    _, _, phi = R.sphere(n, DX, np.asarray(center) - origin, radius)
    hdr = SdfHeader()
    hdr.ni = hdr.nj = hdr.nk = n[0]
    hdr.h = DX
    return sdf.LevelSet(hdr, np.ascontiguousarray(phi.reshape(-1))), tuple(origin), (2 * m * DX,) * 3


def kernel_ms(prof, reps):
    out = {"classify": 0.0, "count": 0.0, "write": 0.0}
    for e in prof.key_averages():
        t = (getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)) / 1e3 / reps
        if "SdfClassify" in e.key:
            out["classify"] += t
        elif "sdf_count_kernel" in e.key:
            out["count"] += t
        elif "sdf_write_kernel" in e.key:
            out["write"] += t
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        raise SystemExit("sdf_bench.py needs a CUDA device")
    import claymore_b200 as cb
    from claymore_b200 import sdf

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE,
                         text=True, check=True)
    print(json.dumps({"gpu": smi.stdout.strip()}))
    cfg = cb.Config(domain_bits=BITS, max_ppc=16)
    torch.cuda.init()

    lattice = [sphere_level_set((cx, 0.5, 0.5), 0.1645) for cx in (0.30, 0.70)]
    random = [sphere_level_set((0.5, 0.5, 0.5), 0.207)]
    for name, bodies, mode in (("lattice_two_spheres", lattice, "lattice"), ("random_sphere", random, "random")):
        counts = [len(sdf.sample(ls, cfg, off, span, ppc=8, mode=mode)) for ls, off, span in bodies]   # warm-up
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                for ls, off, span in bodies:
                    sdf.sample(ls, cfg, off, span, ppc=8, mode=mode)
        ms = kernel_ms(prof, args.reps)
        nodes = sum(ls.phi.size for ls, _, _ in bodies)
        # classify reads every node once; count and write read phi through L2 (the algorithmic bytes count it once)
        alg = 4 * nodes + 12 * sum(counts)
        total = ms["classify"] + ms["count"] + ms["write"]
        print(json.dumps({"workload": name, "particles": sum(counts), "level_set_nodes": nodes, "kernel_ms": {k: round(v, 4) for k, v in ms.items()},
                          "total_ms": round(total, 4), "alg_bytes": alg, "alg_TBps": round(alg / (total * 1e-3) / 1e12, 3),
                          "share_of_3.35TBps": round(alg / (total * 1e-3) / PEAK_BW, 3)}))

    # host time: init_model_sdf against samplers.sphere + init_model (the two bench spheres, one simulator each)
    res = {}
    for how in ("sphere+init_model", "init_model_sdf", "sphere+init_model", "init_model_sdf"):
        sim = cb.GmpmSimulator(config=cfg, max_blocks=120000)
        t0 = time.perf_counter()
        for cx, (ls, off, span) in zip((0.30, 0.70), lattice):
            if how == "init_model_sdf":
                sim.init_model_sdf(cb.FIXED_COROTATED, ls, off, span, ppc=8, mode="lattice")
            else:
                sim.init_model(cb.FIXED_COROTATED, cb.samplers.sphere(DX, (cx, 0.5, 0.5), 0.1645))
        sim.sync()
        res.setdefault(how, []).append(round(time.perf_counter() - t0, 3))
        res.setdefault(how + "_particles", sum(sim.counts))
        sim.close()
    print(json.dumps({"host_time_s": res}))


if __name__ == "__main__":
    main()
