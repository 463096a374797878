#!/usr/bin/env python
"""Where a g2p2g CTA spends its cycles, phase by phase, on bench.py workloads (one GPU):
    python tools/g2p2g_phase_clocks.py [--workloads spheres40m,sand20m,fluid40m] [--steps 50] [--warmup 5] [--lib-dir DIR]
Builds the library with the kernel's per-phase cycle counters switched on (make EXTRA=-DCB200_G2P2G_PHASE_CLOCKS) into a
temporary directory (or --lib-dir), then for every workload runs, in one child process per build, `steps` sub-steps after the
warm-up as plain stream launches: the instrumented build reports thread 0's clock64() intervals of every CTA (g2p2g.cuh,
G2P2GClock), both builds report g2p2g's device time from the step driver's event pairs, so the cost of the counters is stated
beside the shares (`probe_cost` flags a difference above 3 %).
Prints JSON lines: the GPU (name, power limit, max SM clock, SM clock sampled while the steps run), then one line per workload
with every phase's share of all CTA cycles and its cycles per particle block.  Needs a GPU: without one it fails."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PHASES = ["prologue", "phase1", "phase2", "phase3", "flush", "chunk_prologue"]  # G2P2GClock order; then the late-first count and the total
N_CLOCKS = 8
PROBE_TOLERANCE = 0.03


def smi(fields):
    out = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True, check=True)
    return out.stdout.strip().splitlines()[0]


def child(args):
    """one workload on one build: g2p2g ms per sub-step and (instrumented) the cycle sums"""
    sys.path.insert(0, ROOT)
    import ctypes as C
    from claymore_b200 import _capi
    _capi._LIB = args.lib
    import torch
    from claymore_b200 import scenes
    if not torch.cuda.is_available():
        raise SystemExit("g2p2g_phase_clocks.py needs a CUDA device: nothing was measured")
    scene = scenes.workload(args.run)[0]
    max_ppc = 32 if args.run.startswith("mixed") else 128   # bench.py's rule
    L = _capi.lib()
    probe = getattr(L, "cb200_g2p2g_phase_clocks", None)
    if args.instrumented and probe is None:
        raise SystemExit(f"{args.lib} does not export cb200_g2p2g_phase_clocks: not an instrumented build")
    clocks = (C.c_ulonglong * N_CLOCKS)()
    stream = torch.cuda.Stream()
    sim = scenes.build_engine(scene, dt=1e-4, max_blocks=scenes.max_blocks_for(scene), max_ppc=max_ppc, stream=stream.cuda_stream, auto_grow=False)
    sim.step(args.warmup)
    sim.sync()
    sim.profile(True)
    sim.step(2)
    sim.sync()
    sim.profile_phases(), sim.profile_read()
    if probe is not None:
        _capi.check(probe(clocks, 1), "phase clocks reset")
    sim.step(args.steps)
    sm_clock = smi("clocks.sm")   # sampled while the enqueued sub-steps run
    sim.sync()
    sim.profile_phases()
    g2p2g_ms, launches = sim.profile_read()
    sim.profile(False)
    if probe is not None:
        _capi.check(probe(clocks, 0), "phase clocks read")
    st = sim.stats()
    sim.close()
    assert st.error == 0, f"engine error bits {st.error}"
    print(json.dumps({"g2p2g_ms_per_step": g2p2g_ms / args.steps, "launches": launches, "pbc": st.particle_block_count,
                      "sm_clock": sm_clock, "clocks": list(clocks) if probe is not None else None}))


def run_child(workload, lib, instrumented, args):
    cmd = [sys.executable, os.path.abspath(__file__), "--run", workload, "--lib", lib, "--steps", str(args.steps), "--warmup", str(args.warmup)]
    if instrumented:
        cmd.append("--instrumented")
    out = subprocess.run(cmd, stdout=subprocess.PIPE, text=True, check=True).stdout
    return json.loads(out.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="spheres40m,sand20m,fluid40m")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--lib-dir", default=None, help="where the instrumented library is built (default: a temporary directory)")
    ap.add_argument("--run", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--lib", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--instrumented", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.run:
        return child(args)

    lib_dir = args.lib_dir or tempfile.mkdtemp(prefix="cb200_phase_clocks_")
    probe_lib = os.path.join(lib_dir, "libclaymore_b200.so")
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "claymore_b200", "csrc"), "-s", "EXTRA=-DCB200_G2P2G_PHASE_CLOCKS", f"OUT={probe_lib}"])
    default_lib = os.path.join(ROOT, "claymore_b200", "lib", "libclaymore_b200.so")
    if not os.path.exists(default_lib):
        raise SystemExit(f"{default_lib} not found: build the library first (__graft_entry__.build())")
    name, power, max_clock = [s.strip() for s in smi("name,power.limit,clocks.max.sm").split(",")]
    print(json.dumps({"gpu": name, "power_limit": power, "max_sm_clock": max_clock}))

    for wl in [w for w in args.workloads.split(",") if w]:
        base = run_child(wl, default_lib, False, args)
        inst = run_child(wl, probe_lib, True, args)
        c = inst["clocks"]
        total = c[7]
        blocks = inst["pbc"] * args.steps   # particle blocks of the timed sub-steps (block count of the last one)
        line = {"workload": wl, "steps": args.steps, "particle_blocks_per_step": inst["pbc"], "sm_clock": inst["sm_clock"],
                "g2p2g_ms_per_step": round(base["g2p2g_ms_per_step"], 4), "g2p2g_ms_per_step_instrumented": round(inst["g2p2g_ms_per_step"], 4)}
        cost = inst["g2p2g_ms_per_step"] / base["g2p2g_ms_per_step"] - 1.0
        line["probe_cost"] = round(cost, 4)
        if abs(cost) > PROBE_TOLERANCE:
            line["note"] = f"the counters change g2p2g's time by {100 * cost:+.1f} %: read the shares with that in mind"
        line["share_of_cta_cycles"] = {p: round(c[i] / total, 4) for i, p in enumerate(PHASES)}
        line["share_of_cta_cycles"]["unattributed"] = round(1.0 - sum(c[:6]) / total, 4)
        line["cycles_per_block"] = {p: round(c[i] / blocks, 1) for i, p in enumerate(PHASES)}
        line["blocks_first_model_not_0_per_step"] = round(c[6] / args.steps, 1)
        line["prologue_and_chunk_prologue_share"] = round((c[0] + c[5]) / total, 4)
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
