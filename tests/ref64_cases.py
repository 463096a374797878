"""The scene matrix of the float64-reference tests (test_ref64_cpu.py, test_gpu_ref64.py) and its builders.

A case is dict(domain_bits, models=[dict(material, pos, v0, rho, vol, args)], dt, steps, cfl, max_ppc): ``args`` are the
material setter's arguments after (rho, vol); ``steps`` the sub-steps k at which one sub-step is checked.
"""
import numpy as np

import ref64
from claymore_b200 import samplers
from claymore_b200._capi import Config

J_FLUID, FIXED_COROTATED, SAND, NACC = ref64.J_FLUID, ref64.FIXED_COROTATED, ref64.SAND, ref64.NACC
SETTER = {J_FLUID: "update_j_fluid_parameters", FIXED_COROTATED: "update_fr_parameters", SAND: "update_sand_parameters", NACC: "update_nacc_parameters"}
DEFAULT_ARGS = {J_FLUID: (4e4, 7.15, 0.01), FIXED_COROTATED: (5e3, 0.4), SAND: (5e3, 0.4), NACC: (5e3, 0.4, 0.5, 0.8)}


def model(material, pos, v0, dx, rho=1e3, vol=None, args=None):
    return dict(material=material, pos=np.ascontiguousarray(pos, np.float32), v0=tuple(float(v) for v in v0), rho=rho,
                vol=dx ** 3 / 8 if vol is None else vol, args=DEFAULT_ARGS[material] if args is None else tuple(args))


def ref_params(m):
    return ref64.params(m["material"], m["rho"], m["vol"], *m["args"])


def box(dx, lo, hi):
    return samplers.uniform_box(dx, lo, hi)


def _case(domain_bits, models, steps, dt=1e-4, cfl=0.5, max_ppc=128, **kw):
    return dict(domain_bits=domain_bits, models=models, steps=steps, dt=dt, cfl=cfl, max_ppc=max_ppc, **kw)


def _cube(material, domain_bits=6, lo=20, hi=32, v0=(0.3, -1.0, 0.2), **kw):
    dx = 1.0 / (1 << domain_bits)
    return _case(domain_bits, [model(material, box(dx, (lo,) * 3, (hi,) * 3), v0, dx)], **kw)


def _walls(material):
    """A 4^3-cell cube pressed into each of the six wall bands and one into a corner (64^3 grid, bands: cells < 8, >= 56)."""
    dx = 1.0 / 64
    ms = []
    for axis in range(3):
        for lo, v in ((3, -1.0), (57, 1.0)):
            a, b = [28] * 3, [32] * 3
            a[axis], b[axis] = lo, lo + 4
            v0 = [0.0] * 3
            v0[axis] = v
            ms.append(model(material, box(dx, a, b), v0, dx))
    ms.append(model(material, box(dx, (3, 3, 3), (7, 7, 7)), (-1.0, -1.0, -1.0), dx))
    return _case(6, ms, [0, 3])


def _multi_model():
    """kMaxModels = 8 models: three FIXED_COROTATED models with different rho, volume, E, nu interleaved in one cube (they share
    particle blocks), two fluids with different bulk moduli, sand, NACC and a one-particle FIXED_COROTATED model."""
    dx = 1.0 / 64
    cube = box(dx, (20, 20, 20), (28, 28, 28))
    v0 = (0.5, -1.0, 0.3)
    ms = [model(FIXED_COROTATED, cube[i::3], v0, dx, rho=r, vol=vf * dx ** 3 / 8, args=a)
          for i, (r, vf, a) in enumerate(((1e3, 1.0, (5e3, 0.4)), (2.5e3, 0.6, (2e4, 0.3)), (400.0, 1.7, (1e3, 0.2))))]
    ms.append(model(J_FLUID, box(dx, (34, 20, 20), (40, 26, 26)), (-0.5, -1.0, 0.0), dx))
    ms.append(model(J_FLUID, box(dx, (34, 30, 20), (40, 36, 26)), (-0.5, 0.5, 0.0), dx, rho=800.0, args=(1e5, 7.0, 0.05)))
    ms.append(model(SAND, box(dx, (20, 32, 20), (26, 38, 26)), (0.0, -1.0, 0.0), dx))
    ms.append(model(NACC, box(dx, (20, 20, 32), (26, 26, 38)), (0.0, 0.0, -1.0), dx, rho=1.5e3, args=(1e4, 0.3, 0.4, 1.0)))
    ms.append(model(FIXED_COROTATED, np.array([[30.3 * dx, 40.1 * dx, 30.7 * dx]]), (1.0, 0.0, 0.0), dx, rho=3e3, args=(1e4, 0.25)))
    return _case(6, ms, [0, 3], max_near_branch=0.25)   # the sand model starts on the cone tip (F = I)


def _floor(material, steps):
    """A column standing in the floor wall band (cells y < 8): the floor stops it and the material is compressed."""
    dx = 1.0 / 64
    return _case(6, [model(material, box(dx, (26, 3, 26), (34, 15, 34)), (0.0, -2.0, 0.0), dx)], steps)


def _block_sizes():
    """Particle blocks holding 1, 31, 32, 33, 511, 512, 513 and 1024 particles (the bin and chunk edges of g2p2g and the
    rebuild), and a one-particle model."""
    dx = 1.0 / 128
    rng = np.random.default_rng(5)
    pts = []
    for i, n in enumerate((1, 31, 32, 33, 511, 512, 513, 1024)):
        b = np.array([4 + 4 * (i % 4), 8 + 8 * (i // 4), 12])
        lo = (4 * b + 2 - 0.45) * dx
        pts.append(rng.uniform(lo, lo + 3.9 * dx, (n, 3)))
    one = np.array([[64.2 * dx, 64.7 * dx, 40.4 * dx]])
    return _case(7, [model(FIXED_COROTATED, np.concatenate(pts), (0.4, -0.7, 0.2), dx), model(J_FLUID, one, (0.0, -1.0, 0.0), dx)], [0, 3])


def _high_faces():
    """Particles at cell index 4G - 1 and 4G (within 1.5 dx of the top faces) of all three axes and in the top corner: their
    stencils reach node 4G, which does not exist, and what they would add there is dropped (64^3 grid, 4G = 64)."""
    dx = 1.0 / 64
    top = np.array([62.8, 63.1, 63.6, 64.2])                  # cell index 63, 63, 64, 64
    mid = np.array([30.25, 30.75, 31.25, 31.75])
    ms = []
    for axis in range(3):
        ax = [mid, mid, mid]
        ax[axis] = top
        ms.append(np.stack(np.meshgrid(*ax, indexing="ij"), -1).reshape(-1, 3))
    ms.append(np.stack(np.meshgrid(top, top, top, indexing="ij"), -1).reshape(-1, 3))
    return _case(6, [model(FIXED_COROTATED, np.concatenate(ms) * dx, (0.5, 0.5, 0.5), dx)], [0, 2])


CASES = {
    "fc_cube": _cube(FIXED_COROTATED, steps=[0, 3]),
    "fluid_cube": _cube(J_FLUID, steps=[0, 3]),
    "sand_cube": _cube(SAND, steps=[0, 3], max_near_branch=1.0),   # F = I: every particle sits on the cone tip (sand_floor is off it)
    "nacc_cube": _cube(NACC, steps=[0, 3]),
    "walls": _walls(FIXED_COROTATED),
    "walls_fluid": _walls(J_FLUID),
    "multi_model_8": _multi_model(),
    "cfl_bound": _cube(FIXED_COROTATED, v0=(1.0, -10.0, 0.5), dt=1e-3, steps=[0, 4]),
    # fps = 390: a frame is 25.6 sub-steps of 1e-4, so sub-step 25 ends the frame with new_dt = 0.64 dt (the stress term's dt)
    "fc_floor_frame_end": dict(_floor(FIXED_COROTATED, [24, 25, 26]), fps=390),
    # a fluid slab slammed into the floor band at 45 m/s: the CFL-bound sub-steps compress it to the J clamp (quirk #6) by sub-step 2
    "fluid_clamp": _case(6, [model(J_FLUID, box(1.0 / 64, (26, 8, 26), (34, 14, 34)), (0.0, -45.0, 0.0), 1.0 / 64)], [1, 2], dt=1e-3, cfl=0.7,
                         max_near_branch=0.05),
    "sand_floor": dict(_floor(SAND, [30, 60]), max_near_branch=0.1),
    "nacc_floor": dict(_floor(NACC, [30, 60]), max_near_branch=0.1),
    "fluid_floor": _floor(J_FLUID, [30, 60]),
    # two NACC slabs sliding past each other: the shear takes the particles at the interface to the yield surface (projection
    # with hardening)
    "nacc_shear": _case(6, [model(NACC, box(1.0 / 64, (24, 20, 24), (36, 26, 36)), (2.0, 0.0, 0.0), 1.0 / 64),
                            model(NACC, box(1.0 / 64, (24, 26, 24), (36, 32, 36)), (-2.0, 0.0, 0.0), 1.0 / 64)], [5]),
    "domain_bits_4": _cube(FIXED_COROTATED, domain_bits=4, lo=5, hi=11, steps=[0, 2]),
    "domain_bits_5": _cube(J_FLUID, domain_bits=5, lo=10, hi=20, steps=[0, 2]),
    "domain_bits_10": _cube(FIXED_COROTATED, domain_bits=10, lo=500, hi=508, steps=[0, 2]),
    "max_ppc_8": _cube(FIXED_COROTATED, max_ppc=8, steps=[0, 3]),
    "max_ppc_16": _cube(J_FLUID, max_ppc=16, steps=[0, 3]),
    "max_ppc_64": _cube(NACC, max_ppc=64, steps=[0, 3]),
    "high_faces": _high_faces(),
    "block_sizes": _block_sizes(),
}


class OracleClock:
    """The reference's frame loop around the oracle (gmpm_simulator.cuh:324): the time left in the frame bounds the next dt."""

    def __init__(self, sim):
        self.sim, self.t = sim, np.float32(0.0)

    def time_left(self):
        return float(self.sim.frame - self.t) if self.sim.frame is not None else np.inf

    def step(self, n=1):
        for _ in range(n):
            self.sim.step(1, time_left=self.time_left() if self.sim.frame is not None else 1e30)
            self.t = np.float32(self.t + np.float32(self.sim.dt))
            if self.sim.frame is not None and self.t >= self.sim.frame:
                self.t = np.float32(0.0)


def engine_time_left(sim, case):
    """The frame's time left as the engine's clock sees it (frame_time - step_time in float32)."""
    if not case.get("fps"):
        return np.inf
    return float(np.float32(1.0 / case["fps"]) - np.float32(sim.stats().step_time))


# ---- kernel-level inputs: the oracle's containers, with deformation gradients the pipeline rarely produces ---------------
def _rot(a, b, c):
    ca, sa, cb, sb, cc, sc = np.cos(a), np.sin(a), np.cos(b), np.sin(b), np.cos(c), np.sin(c)
    return (np.array([[ca, -sa, 0], [sa, ca, 0], [0, 0, 1]]) @ np.array([[cb, 0, sb], [0, 1, 0], [-sb, 0, cb]])
            @ np.array([[1, 0, 0], [0, cc, -sc], [0, sc, cc]]))


def extreme_f(n, seed=0):
    """n deformation gradients, column-major rows: a quarter compressed to det F ~ 0.1, a quarter inverted (det < 0), a
    quarter nearly singular (smallest singular value 1e-5), a quarter stretched and sheared."""
    rng = np.random.default_rng(seed)
    out = np.empty((n, 9))
    for i in range(n):
        R1, R2 = _rot(*rng.uniform(0, 2 * np.pi, 3)), _rot(*rng.uniform(0, 2 * np.pi, 3))
        kind = i % 4
        s = {0: rng.uniform(0.44, 0.48, 3), 1: rng.uniform(0.7, 1.2, 3) * np.array([1, 1, -1]),
             2: np.array([1.0, 1.0, 1e-5]) * rng.uniform(0.9, 1.1, 3), 3: rng.uniform(0.8, 1.4, 3)}[kind]
        F = R1 @ np.diag(s) @ R2
        out[i] = F.T.reshape(9)
    return out.astype(np.float32)


def kernel_level_inputs(ob, material, deform=False, steps=4):
    """The oracle after ``steps`` sub-steps of a small cube, its grid turned into velocities by the oracle's grid update, and
    with deform=True the current bins' F replaced by extreme_f (the oracle's particle_state then reads them back)."""
    case = _cube(material, steps=[steps])
    osim = build_oracle(ob, case)
    osim.step(steps)
    cur = osim.buffer_arrays(0, 0)
    if deform:
        bins = cur["bins"].reshape(-1, 512)
        F = extreme_f(32 * len(bins)).reshape(len(bins), 32, 9)
        for d in range(9):
            bins[:, (3 + d) * 32:(4 + d) * 32] = F[:, :, d]
    return case, osim


def states_from_bins(bins, offsets, sizes, block_count, material):
    """Particle rows of the bins of ``block_count`` blocks (bucket order)."""
    nch, bf = ref64.CHANNELS[material], (128 if material == J_FLUID else 512)
    rows = []
    for b in range(block_count):
        n = int(sizes[b])
        for bi in range((n + 31) // 32):
            o = (int(offsets[b]) + bi) * bf
            rows.append(bins[o:o + nch * 32].reshape(nch, 32)[:, :min(32, n - 32 * bi)].T)
    return np.concatenate(rows) if rows else np.zeros((0, nch), np.float32)


def config(case):
    return Config(domain_bits=case["domain_bits"], max_ppc=case["max_ppc"], cfl=case["cfl"])


def build_oracle(ob, case, max_blocks=6000):
    cfg = ob.make_config(domain_bits=case["domain_bits"], max_ppc=case["max_ppc"], cfl=case["cfl"])
    sim = ob.OracleSim(cfg, case["dt"], max_blocks)
    sim.frame = np.float32(1.0 / case["fps"]) if case.get("fps") else None
    for m in case["models"]:
        mid = sim.init_model(m["material"], m["pos"], m["v0"])
        getattr(sim, SETTER[m["material"]])(mid, m["rho"], m["vol"], *m["args"])
    sim.initial_setup()
    return sim


def build_engine(case, use_graph=True, max_blocks=6000):
    from claymore_b200.simulator import GmpmSimulator
    sim = GmpmSimulator(dt=case["dt"], fps=case.get("fps", 0), config=config(case), max_blocks=max_blocks, use_graph=use_graph)
    for m in case["models"]:
        mid = sim.init_model(m["material"], m["pos"], m["v0"])
        getattr(sim, SETTER[m["material"]])(m["rho"], m["vol"], *m["args"], model=mid)
    sim.initial_setup()
    return sim
