"""Cost of the signed-distance collider on the bench's flagship workload.

Runs the 40 M-particle two-sphere scene (bench.py's default, 512^3 grid) with a static sticky floor box under the spheres and
with no collider, alternating the two in one process, and prints JSON lines: the GPU (name, power limit, max SM clock), then per
run the sub-step time (CUDA events, graph replay) and the per-phase milliseconds of profile_phases (grid_update first).

    python tools/collider_bench.py [--steps 50] [--warmup 10] [--rounds 3]

--objects compares, in alternating rounds, no collider, the level-set floor, the same floor as one analytic box, and 4 and 16
analytic objects (the floor box, then spheres and cylinders off to the sides of the spheres, and planes below the floor).  Each
run also reports the grid update's kernel time per sub-step from torch.profiler (a run of its own) and the device memory the
collider or the objects add (free memory before and after they are set).

    python tools/collider_bench.py --objects [--steps 50] [--warmup 10] [--rounds 3]

--levelsets compares, in alternating rounds, no collider, the dense level-set floor, the analytic floor box, the same floor as a
level-set collision object (a box level set on a lattice of node spacing dx, two cells wider than the floor on every side), and a
dragon-shaped obstacle (two_dragons.sdf's 77 x 118 x 401 nodes, two ellipsoids, at node spacing dx) through the spheres' lower
halves, with the grid update's kernel time and the device memory each adds, as --objects.

    python tools/collider_bench.py --levelsets [--steps 50] [--warmup 10] [--rounds 3]

--forces compares, in alternating rounds, the boundary impulse report off and on (GmpmSimulator.report_forces, DESIGN.md
section 2.13) for the level-set floor, the analytic floor box and 4 and 16 analytic objects, with the grid update's kernel time.

    python tools/collider_bench.py --forces [--steps 50] [--warmup 10] [--rounds 3]

--tracks compares, in alternating rounds, the analytic floor box and 4 and 16 analytic objects untracked against the same objects each
on a smooth motion track (DESIGN.md section 2.14; a slow drift and turn, so that the scene stays the same), with the grid update's
kernel time.

    python tools/collider_bench.py --tracks [--steps 50] [--warmup 10] [--rounds 3]
"""
import ctypes as C
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def run(scene, field, args, stream, objs=None, forces=False):
    import torch
    from claymore_b200 import scenes
    sim = scenes.build_engine(scene, dt=args.dt, max_blocks=scenes.max_blocks_for(scene), stream=stream.cuda_stream, auto_grow=False)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    if field is not None:
        sim.set_collider(field[0], field[1], type="sticky")
    if objs:
        sim.set_collision_objects(objs)
    if forces:
        sim.report_forces(True)
    torch.cuda.synchronize()
    added = free0 - torch.cuda.mem_get_info()[0]
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
    kernel_ms = None
    if args.objects or args.levelsets or args.forces or args.tracks:
        from torch.profiler import ProfilerActivity, profile
        sim.sync()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            sim.step(args.steps)
            sim.sync()
        us = sum(e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total for e in prof.key_averages() if "grid_update" in e.key)
        kernel_ms = round(us / 1000.0 / args.steps, 4)
    st = sim.stats()
    sim.close()
    assert st.error == 0, f"engine error bits {st.error}"
    return {"substep_ms": round(substep_ms, 4), "phases_ms": phases, "grid_update_kernel_ms": kernel_ms, "added_device_bytes": added}


def object_sets(top):
    """the analytic variants of --objects: the floor box alone, 4 and 16 objects (the floor first)"""
    from claymore_b200 import objects
    floor = objects.box((0.1, 0.1, 0.1), (0.9, top, 0.9), type="sticky")
    extra = []
    for i in range(15):
        k = i % 3
        if k == 0:
            extra.append(objects.sphere((0.12 + 0.05 * i, 0.75, 0.12), 0.03, type="slip", friction=0.3))
        elif k == 1:
            extra.append(objects.cylinder((0.88, 0.6, 0.12 + 0.05 * i), 0.03, 0.1, type="separate", friction=0.3, omega=(0.0, 1.0, 0.0)))
        else:
            extra.append(objects.plane((0.5, 0.1 - 0.005 * i, 0.5), (0.0, 1.0, 0.0), type="slip"))
    return {"analytic_floor": [floor], "objects4": [floor] + extra[:3], "objects16": [floor] + extra}


def tracked(objs):
    """copies of objs, each on a three-key smooth track from its rest pose (a drift of 1e-3 and a turn of 0.01 rad per second);
    omega, the one velocity object_sets gives, is dropped (a tracked object moves only along its track)"""
    from claymore_b200 import objects
    from claymore_b200._capi import CollisionObject
    out = []
    for o in objs:
        c = CollisionObject.from_buffer_copy(o)
        c.omega[:] = [0.0, 0.0, 0.0]
        p = list(c.trans)
        c.track = objects.track([(0.0, p, (1, 0, 0, 0)), (1.0, [p[0], p[1] + 1e-3, p[2]], (0.99999, 0.0, 0.005, 0.0)),
                                 (2.0, [p[0] + 1e-3, p[1] + 1e-3, p[2]], (0.99995, 0.0, 0.01, 0.0))], "smooth")
        out.append(c)
    return out


def _level_set(phi, h):
    """an sdf.LevelSet of phi[k, j, i] with node spacing h"""
    import numpy as np
    from claymore_b200 import sdf
    from claymore_b200._capi import SdfHeader
    nk, nj, ni = phi.shape
    return sdf.LevelSet(SdfHeader(ni, nj, nk, (C.c_float * 3)(0, 0, 0), h), np.ascontiguousarray(phi, np.float32).reshape(-1))


def levelset_sets(top, dx):
    """the level-set variants of --levelsets: the floor box as a level-set object, and the dragon-shaped obstacle"""
    import numpy as np
    from claymore_b200 import objects
    lo, hi = np.array([0.1, 0.1, 0.1]), np.array([0.9, top, 0.9])
    org = lo - 2 * dx
    n = np.floor((hi + 2 * dx - org) / dx).astype(int) + 1
    x = (org[0] + dx * np.arange(n[0]))[None, None, :]
    y = (org[1] + dx * np.arange(n[1]))[None, :, None]
    z = (org[2] + dx * np.arange(n[2]))[:, None, None]
    phi = np.maximum(np.maximum(np.maximum(lo[0] - x, x - hi[0]), np.maximum(lo[1] - y, y - hi[1])), np.maximum(lo[2] - z, z - hi[2]))
    floor = objects.levelset(_level_set(phi, dx), org, (n - 1) * dx, type="sticky")
    dn = (77, 118, 401)
    L = [(d - 1) * dx for d in dn]
    x = (dx * np.arange(dn[0]))[None, None, :]
    y = (dx * np.arange(dn[1]))[None, :, None]
    z = (dx * np.arange(dn[2]))[:, None, None]
    a = np.sqrt(((x - 0.5 * L[0]) / (0.4 * L[0])) ** 2 + ((y - 0.45 * L[1]) / (0.4 * L[1])) ** 2 + ((z - 0.25 * L[2]) / (0.2 * L[2])) ** 2) - 1
    b = np.sqrt(((x - 0.5 * L[0]) / (0.35 * L[0])) ** 2 + ((y - 0.55 * L[1]) / (0.4 * L[1])) ** 2 + ((z - 0.72 * L[2]) / (0.22 * L[2])) ** 2) - 1
    dragon = objects.levelset(_level_set(np.minimum(a, b) * min(L) * 0.2, dx), (0.5 - 0.5 * L[0], top - 0.05, 0.5 - 0.5 * L[2]),
                              [v + 1e-9 for v in L], type="slip", friction=0.3)
    return {"levelset_floor": [floor], "dragon": [dragon]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--dt", type=float, default=1e-4)
    ap.add_argument("--objects", action="store_true", help="also the analytic floor box, 4 and 16 analytic objects")
    ap.add_argument("--levelsets", action="store_true", help="also the analytic floor box, the floor as a level-set object and a dragon")
    ap.add_argument("--forces", action="store_true", help="the impulse report off and on: level-set floor, analytic floor, 4 and 16 objects")
    ap.add_argument("--tracks", action="store_true", help="untracked against tracked: analytic floor, 4 and 16 objects")
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
    sets = object_sets(top) if args.objects else {}
    if args.levelsets:
        sets = {"analytic_floor": object_sets(top)["analytic_floor"], **levelset_sets(top, 1.0 / (1 << scene["domain_bits"]))}
    if args.forces:
        sets = object_sets(top)
        names = [(n, f) for n in ["floor"] + sorted(sets) for f in (False, True)]
        for r in range(args.rounds):
            for name, forces in (names if r % 2 == 0 else names[::-1]):
                res = run(scene, field if name == "floor" else None, args, stream, sets.get(name), forces=forces)
                print(json.dumps({"round": r, "collider": name, "forces": forces, "steps": args.steps, **res}), flush=True)
        return
    if args.tracks:
        sets = object_sets(top)
        names = [(n, t) for n in sorted(sets) for t in (False, True)]
        for r in range(args.rounds):
            for name, tr in (names if r % 2 == 0 else names[::-1]):
                res = run(scene, None, args, stream, tracked(sets[name]) if tr else sets[name])
                print(json.dumps({"round": r, "collider": name, "tracks": tr, "steps": args.steps, **res}), flush=True)
        return
    names = ["floor", "none"] + sorted(sets)
    for r in range(args.rounds):
        order = names if r % 2 == 0 else names[::-1]
        for name in order:
            res = run(scene, field if name == "floor" else None, args, stream, sets.get(name))
            print(json.dumps({"round": r, "collider": name, "steps": args.steps, **res}), flush=True)


if __name__ == "__main__":
    main()
