"""Cost of checkpoint / restore on the bench's flagship workload (40 M-particle two spheres, 512^3 grid, a ~1.9 GB blob).

Prints JSON lines: the GPU (name, power limit, SM clock), then
  * the snapshot gather kernel's time (torch.profiler's CUPTI kernel records) and its bytes/s against the 3.35 TB/s data-sheet
    bandwidth (bytes = blob read + blob written), the host time of checkpoint_begin and the wait in checkpoint_end;
  * the time of 2 x --every sub-steps (CUDA events) with one overlapped checkpoint between the halves (begin, the next
    sub-steps, end) against none, in alternating runs that each restart from the same restored state;
  * the restore time, and an exact round-trip check at this size: the checkpoint of the restored simulator equals the original
    once canonically ordered (rows compared as a sorted multiset of 64-bit row hashes, header, keys and grid bit for bit).

    python tools/checkpoint_bench.py [--every 417] [--rounds 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK_BW = 3.35e12  # H100 SXM HBM3 data sheet


def _row_hashes(state):
    """order-free fingerprint of the rows of a [n, C] float32 array: one 64-bit hash per row, sorted"""
    u = state.view(np.uint32).astype(np.uint64)
    h = np.zeros(len(state), np.uint64)
    for c in range(state.shape[1]):
        h = (h ^ u[:, c]) * np.uint64(0x100000001B3 + 2 * c)
        h ^= h >> np.uint64(29)
    return np.sort(h)


def _canonical(blob):
    from claymore_b200 import checkpoint, scenes
    d = checkpoint.read(blob)
    o = np.argsort(scenes.key_hash(d["keys"]))
    head = {k: v for k, v in d.items() if k not in ("states", "keys", "grid")}
    return head, [_row_hashes(s) for s in d["states"]], d["keys"][o], d["grid"][o]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--every", type=int, default=417, help="sub-steps between checkpoints (one frame at 24 fps and dt 1e-4)")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--dt", type=float, default=1e-4)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("checkpoint_bench.py needs a CUDA device")
    from claymore_b200 import scenes
    from claymore_b200.simulator import GmpmSimulator

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv"], stdout=subprocess.PIPE, text=True, check=True)
    print(json.dumps({"gpu": smi.stdout.strip().splitlines()}), flush=True)
    scene = scenes.workload("spheres40m")[0]
    stream = torch.cuda.Stream()
    sim = scenes.build_engine(scene, dt=args.dt, max_blocks=scenes.max_blocks_for(scene), stream=stream.cuda_stream, auto_grow=False)
    sim.step(args.warmup)
    sim.sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def kernel_ms(prof, name):
        return sum(getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0) for e in prof.key_averages() if name in e.key) / 1e3

    # snapshot kernel (CUPTI kernel times), host time of begin, wait in end with nothing to overlap
    from torch.profiler import ProfilerActivity, profile
    for rep in range(3):
        sim.sync()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            t0 = time.perf_counter()
            nbytes = sim.checkpoint_begin()
            t1 = time.perf_counter()
            sim.checkpoint_end()
            t2 = time.perf_counter()
        snap, scan = kernel_ms(prof, "snapshot_kernel"), kernel_ms(prof, "scan_kernel")
        moved = 2 * (nbytes - 1024)
        print(json.dumps({"snapshot": rep, "blob_bytes": nbytes, "snapshot_kernel_ms": round(snap, 3), "scan_kernels_ms": round(scan, 3),
                          "achieved_TBps": round(moved / (snap * 1e-3) / 1e12, 3) if snap else None,
                          "fraction_of_3.35TBps": round(moved / (snap * 1e-3) / PEAK_BW, 3) if snap else None,
                          "begin_host_ms": round((t1 - t0) * 1e3, 3), "end_wait_ms_no_overlap": round((t2 - t1) * 1e3, 3)}), flush=True)

    # every run starts from the same state (restored from one checkpoint): `every` sub-steps, then either a checkpoint whose
    # copy overlaps the next `every` sub-steps or none
    start = sim.save_checkpoint()
    sim.close()
    n = 2 * args.every
    restore_ms = []
    for r in range(args.rounds):
        for mode in (("none", "checkpoint") if r % 2 == 0 else ("checkpoint", "none")):
            run = GmpmSimulator.from_checkpoint(start, stream=stream.cuda_stream, auto_grow=False)
            t = time.perf_counter()
            run.restore(start)
            restore_ms.append((time.perf_counter() - t) * 1e3)
            run.step(2)     # graph replay warm
            run.sync()
            e0.record(stream)
            run.step(args.every)
            wait = None
            if mode == "checkpoint":
                t = time.perf_counter()
                run.checkpoint_begin()
                begin_ms = (time.perf_counter() - t) * 1e3
            run.step(args.every)
            e1.record(stream)
            if mode == "checkpoint":
                t = time.perf_counter()
                run.checkpoint_end()
                wait = (time.perf_counter() - t) * 1e3
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1)
            st = run.stats()
            assert st.error == 0, st.error
            out = {"round": r, "mode": mode, "substeps": n, "ms_total": round(ms, 2), "ms_per_substep": round(ms / n, 4)}
            if mode == "checkpoint":
                out.update(begin_host_ms=round(begin_ms, 3), end_wait_ms=round(wait, 3))
            print(json.dumps(out), flush=True)
            run.close()

    # the exact round trip at this size
    r = GmpmSimulator.from_checkpoint(start, stream=stream.cuda_stream, auto_grow=False)
    r.restore(start)
    again = r.save_checkpoint()
    r.close()
    a, b = _canonical(start), _canonical(again)
    assert a[0] == b[0], "checkpoint header differs after a round trip"
    assert all(np.array_equal(x, y) for x, y in zip(a[1], b[1])), "particle rows differ after a round trip"
    assert a[2].tobytes() == b[2].tobytes() and a[3].tobytes() == b[3].tobytes(), "grid differs after a round trip"
    print(json.dumps({"restore_ms": [round(x, 1) for x in restore_ms], "blob_bytes": len(start), "round_trip": "exact"}), flush=True)


if __name__ == "__main__":
    main()
