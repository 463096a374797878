#!/usr/bin/env python
"""Small driver for compute-sanitizer runs (memcheck / racecheck / synccheck) of the whole sub-step on an H100:
    compute-sanitizer --tool racecheck python tools/sanitize_small.py [scene] [steps]
Scenes: small_cube (one model), two_models, mixed (fluid + sand + fixed-corotated in one partition), checkpoint (mixed: step,
checkpoint, restore into a fresh simulator, step again), output (mixed: step, a frame of .bgeo files with v and J written while
further sub-steps run), sdf (a sphere level set sampled on the device in random and lattice mode, then stepped)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from claymore_b200 import scenes  # noqa: E402


def sdf_engine():
    import numpy as np
    from claymore_b200 import Config, FIXED_COROTATED, GmpmSimulator, J_FLUID, sdf
    from claymore_b200._capi import SdfHeader
    n = 17
    g = np.arange(n, dtype=np.float64) * 0.5
    z, y, x = np.meshgrid(g, g, g, indexing="ij")
    hdr = SdfHeader()
    hdr.ni = hdr.nj = hdr.nk = n
    hdr.h = 0.5
    ls = sdf.LevelSet(hdr, (np.sqrt((x - 4) ** 2 + (y - 4) ** 2 + (z - 4) ** 2) - 3.3).astype(np.float32).reshape(-1))
    sim = GmpmSimulator(config=Config(domain_bits=6), use_graph=False, auto_grow=False, max_blocks=2000)
    sim.init_model_sdf(FIXED_COROTATED, ls, (0.2, 0.2, 0.2), 0.25, (0.5, -1.0, 0.0), ppc=8, mode="random", seed=1)
    sim.init_model_sdf(J_FLUID, ls, (0.5, 0.3, 0.5), 0.25, (0.0, -1.0, 0.0), ppc=27, mode="lattice")
    sim.initial_setup()
    return sim


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else "small_cube"
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    if name == "small_cube":
        scene = scenes.small_cube(v0=(0.5, -3.0, 0.4))
    elif name == "two_models":
        scene = scenes.two_cubes_colliding()
    elif name == "sdf":
        scene = None
    else:
        scene = scenes.mixed_materials(domain_bits=7, edge=10)
    sim = scenes.build_engine(scene, use_graph=False, auto_grow=False) if scene is not None else sdf_engine()
    sim.step(steps)
    sim.sync()
    if name == "checkpoint":
        from claymore_b200.simulator import GmpmSimulator
        blob = sim.save_checkpoint()
        sim.close()
        sim = GmpmSimulator.from_checkpoint(blob, use_graph=False, auto_grow=False)
        sim.restore(blob)
        sim.step(steps)
        sim.sync()
    if name == "output":
        import tempfile
        with tempfile.TemporaryDirectory() as d:
            sim.write_frame(d, 1, ("v", "J"))
            sim.step(steps)
            sim.wait_output()
        sim.sync()
    st = sim.stats()
    print("SANITIZE_RUN", name, steps, sum(sim.counts), st.particle_block_count, st.neighbor_block_count, st.exterior_block_count, "error", st.error)
    sim.close()


if __name__ == "__main__":
    main()
