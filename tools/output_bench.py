"""Cost of the per-frame .bgeo output on the bench's flagship workload (40 M-particle two spheres, 512^3 grid).  Files go to a
temporary directory that is deleted afterwards.

Prints JSON lines: the GPU (name, power limit, SM clock), then per attribute set
  * the gather kernel's time (torch.profiler's CUPTI kernel records) and its bytes/s against the 3.35 TB/s data-sheet bandwidth.  The
    algorithmic bytes are estimates computed here: per particle the tag (4 B), the position (12 B), F (36 B) when J is asked for,
    the record written (16-32 B), plus the scan's 4 B per block and 8 KiB of grid[0] per particle block when v is asked for;
  * write_frame's host time, the device-to-host copy with nothing overlapping, and the file write time;
then the time of --steps sub-steps crossing frame boundaries (every --every sub-steps) with output against the same run without,
in alternating runs that restart from one restored state, with the time write_frame spent waiting for the previous frame
(back-pressure).  First-use allocation of the pinned buffer is reported on its own.

    python tools/output_bench.py [--every 100] [--steps 400] [--rounds 2]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK_BW = 3.35e12  # H100 SXM HBM3 data sheet


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--every", type=int, default=100, help="sub-steps between frame outputs")
    ap.add_argument("--steps", type=int, default=400)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--dt", type=float, default=1e-4)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("output_bench.py needs a CUDA device")
    from torch.profiler import ProfilerActivity, profile

    from claymore_b200 import scenes
    from claymore_b200.simulator import GmpmSimulator

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv"], stdout=subprocess.PIPE, text=True, check=True)
    print(json.dumps({"gpu": smi.stdout.strip().splitlines()}), flush=True)
    tmp = tempfile.mkdtemp(prefix="cb200_output_bench_")
    try:
        scene = scenes.workload("spheres40m")[0]
        n = scenes.n_particles(scene)
        stream = torch.cuda.Stream()
        sim = scenes.build_engine(scene, dt=args.dt, max_blocks=scenes.max_blocks_for(scene), stream=stream.cuda_stream, auto_grow=False)
        sim.step(args.warmup)
        sim.sync()
        t = time.perf_counter()
        sim.write_frame(tmp, 0, ("v", "J"))     # first use: staging and pinned buffers (sized for v and J), writer thread
        sim.wait_output()
        print(json.dumps({"first_use_ms": round((time.perf_counter() - t) * 1e3, 1)}), flush=True)

        def kernel_ms(prof, name):
            return sum(getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0) for e in prof.key_averages() if name in e.key) / 1e3

        pbc = sim.stats().particle_block_count
        for attrs in ((), ("J",), ("v", "J")):
            words = 4 + 3 * ("v" in attrs) + ("J" in attrs)
            moved = n * (4 + 12 + (36 if "J" in attrs else 0) + 4 * words) + pbc * 4 + (pbc * 8192 if "v" in attrs else 0)
            for rep in range(2):
                sim.sync()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    t0 = time.perf_counter()
                    paths = sim.write_frame(tmp, 1, attrs)
                    t1 = time.perf_counter()
                    sim.wait_output()
                    t2 = time.perf_counter()
                k = kernel_ms(prof, "output_kernel")
                copy = kernel_ms(prof, "Memcpy DtoH")
                size = sum(os.path.getsize(p) for p in paths)
                print(json.dumps({"attributes": list(attrs), "rep": rep, "bytes_written": size, "gather_kernel_ms": round(k, 3),
                                  "scan_kernels_ms": round(kernel_ms(prof, "scan_kernel"), 3), "algorithmic_bytes": moved,
                                  "achieved_TBps": round(moved / (k * 1e-3) / 1e12, 3) if k else None,
                                  "fraction_of_3.35TBps": round(moved / (k * 1e-3) / PEAK_BW, 3) if k else None,
                                  "write_frame_host_ms": round((t1 - t0) * 1e3, 3), "d2h_ms": round(copy, 1),
                                  "copy_and_write_ms": round((t2 - t1) * 1e3, 1)}), flush=True)
        start = sim.save_checkpoint()
        sim.close()

        for r in range(args.rounds):
            for mode in (("none", "output") if r % 2 == 0 else ("output", "none")):
                run = GmpmSimulator.from_checkpoint(start, stream=stream.cuda_stream, auto_grow=False)
                run.restore(start)
                run.step(2)
                run.sync()
                if mode == "output":    # buffers allocated before the timed window
                    run.write_frame(tmp, 0, ("v", "J"))
                    run.wait_output()
                waits = []
                t = time.perf_counter()
                done = 0
                while done < args.steps:
                    k = min(args.every, args.steps - done)
                    run.step(k)
                    done += k
                    if mode == "output" and done < args.steps:
                        t0 = time.perf_counter()
                        run.write_frame(tmp, done // args.every, ("v", "J"))
                        waits.append((time.perf_counter() - t0) * 1e3)
                run.sync()
                ms = (time.perf_counter() - t) * 1e3
                t = time.perf_counter()
                run.wait_output()
                assert run.stats().error == 0
                out = {"round": r, "mode": mode, "substeps": args.steps, "wall_ms": round(ms, 1), "last_write_wait_ms": round((time.perf_counter() - t) * 1e3, 1)}
                if waits:
                    out["write_frame_ms"] = [round(w, 1) for w in waits]
                print(json.dumps(out), flush=True)
                run.close()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
