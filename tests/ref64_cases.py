"""The scene matrix of the float64-reference tests (test_ref64_cpu.py, test_gpu_ref64.py) and its builders.

A case is dict(domain_bits, models=[dict(material, pos, v0, rho, vol, args)], dt, steps, cfl, max_ppc, gravity, boundary): ``args``
are the material setter's arguments after (rho, vol); ``steps`` the sub-steps k at which one sub-step is checked.  A case with
a ``collider`` = dict(field=(kind, *args), type, friction, rot_mat, trans, trans_vel, omega, dsdt, scale) has a signed-distance
collider (collider_field, collider_struct; the other keys default to SignedDistanceGrid's).  A case with ``objects`` has
analytic collision objects after it (OBJECT_CASES, object_structs).  A case with ``updates`` changes material parameters between
sub-steps (_updated).
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


def _case(domain_bits, models, steps, dt=1e-4, cfl=0.5, max_ppc=128, gravity=-9.8, boundary=2, **kw):
    return dict(domain_bits=domain_bits, models=models, steps=steps, dt=dt, cfl=cfl, max_ppc=max_ppc, gravity=gravity, boundary=boundary, **kw)


def _cube(material, domain_bits=6, lo=20, hi=32, v0=(0.3, -1.0, 0.2), **kw):
    dx = 1.0 / (1 << domain_bits)
    return _case(domain_bits, [model(material, box(dx, (lo,) * 3, (hi,) * 3), v0, dx)], **kw)


def _walls(material, boundary=2):
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
    return _case(6, ms, [0, 3], boundary=boundary)


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


def half_lattice(dx, lo, nudge, n=7, step=3):
    """A sparse n^3 lattice at cell centres (lo + step i + 1/2) dx, in float32.  nudge "exact" keeps them there; "ulp"
    moves every third particle one ulp up and every third one ulp down in all three coordinates, so that cell_index rounds
    the exact ones up, the next ones up and the last ones down.  Below x = 0.5 one ulp is half as long as above it."""
    k = lo + step * np.arange(n) + 0.5
    pos = (np.stack(np.meshgrid(k, k, k, indexing="ij"), -1).reshape(-1, 3) * dx).astype(np.float32)
    if nudge == "ulp":
        i = np.arange(len(pos)) % 3
        pos[i == 1] = np.nextafter(pos[i == 1], np.float32(1))
        pos[i == 2] = np.nextafter(pos[i == 2], np.float32(0))
    return pos


def _half(domain_bits, lo, nudge, v0=(0.0, 0.0, 0.0), gravity=0.0, steps=(0, 1, 2), material=FIXED_COROTATED):
    dx = 1.0 / (1 << domain_bits)
    return _case(domain_bits, [model(material, half_lattice(dx, lo, nudge), v0, dx)], list(steps), gravity=gravity)


def _overflow(material, x_full):
    """Full cells (8 particles each at (c +- 1/4) dx, not over max_ppc = 8) at cell indices x_full .. x_full + 2 and
    y, z = 26 .. 28, and a layer of 4 particles per cell at x = (x_full - 0.53) dx moving at 10 m/s: within one sub-step
    (0.064 dx) the layer crosses the face into the full cells, which then get 12 particles each."""
    dx = 1.0 / 64
    q = np.array([-0.25, 0.25])
    c = np.arange(26, 29)
    yz = np.stack(np.meshgrid((c[:, None] + q).ravel(), (c[:, None] + q).ravel(), indexing="ij"), -1).reshape(-1, 2)
    full = np.concatenate([np.concatenate([np.full((len(yz), 1), x), yz], 1) for x in (np.arange(x_full, x_full + 3)[:, None] + q).ravel()])
    layer = np.concatenate([np.full((len(yz), 1), x_full - 0.53), yz], 1)
    return _case(6, [model(material, np.concatenate([full, layer]) * dx, (10.0, 0.0, 0.0), dx)], [0, 1], max_ppc=8)


# NACC with bm = 0.1 (E 0.12, nu 0.3), beta = 2 and xi = 0.079: p0 = bm (1e-5 + sinh(xi max(-logJp, 0))) starts at 8e-5
# (logJp starts at -0.01), below the 1e-4 under which a projection onto the yield surface skips the hardening update.
# With beta > 1 the other hardening conditions, p_min + 1e-4 < p_trial < p0 - 1e-4, can hold at such a p0: a slight
# tension.  The shear of nacc_shear, with the slabs drawn apart at 2 cm/s, takes particles there at sub-steps 4 and 7.
NACC_SOFT = (0.12, 0.3, 2.0, 0.079)


# ---- material parameters changed between sub-steps ------------------------------------------------------------------------
# A case with ``updates`` = {k: [(scene model, rho, vol, args), ...]} calls the model's material setter right before sub-step k
# (ref64_checks.apply_updates), args in SETTER order after (rho, vol).  Sub-steps k and k + 1 are checked: the two roll parities
# read the parameters of one particle buffer each.  Each update changes one parameter group, on deformed material, so that one
# stale field cannot hide behind another (test_params_cpu.py: ref64 with the parameters before the update is off by 10x its bound).
def _updated(case, updates, steps):
    return dict(case, updates=updates, steps=sorted(set(steps) | {j for k in updates for j in (k, k + 1)}))


def _fc_floor_params():
    c = _floor(FIXED_COROTATED, [])
    v = c["models"][0]["vol"]
    return _updated(c, {20: [(0, 2.5e3, v, (5e3, 0.4))],              # rho: the mass
                        23: [(0, 5e3, v / 2, (5e3, 0.4))],            # vol x 0.5, rho x 2: the same mass, half the stress volume
                        26: [(0, 5e3, v / 2, (2e4, 0.4))],            # E
                        29: [(0, 5e3, v / 2, (2e4, 0.25))]}, [])      # nu


def _fluid_floor_params():
    c = _floor(J_FLUID, [])
    v = c["models"][0]["vol"]
    return _updated(c, {20: [(0, 1e3, v, (1e5, 7.15, 0.01))],         # bulk
                        23: [(0, 1e3, v, (1e5, 3.0, 0.01))],          # gamma
                        26: [(0, 1e3, v, (1e5, 3.0, 10.0))],          # viscosity
                        29: [(0, 1.5e3, v, (1e5, 3.0, 10.0))]}, [])   # rho


def _fluid_clamp_params():
    """fluid_clamp with its viscosity raised at sub-step 1, in the slam.  A change of bulk, gamma or rho there leaves the FP32
    oracle's sub-step 2 within a few percent of the bounds or over them (F, lost particles), and so do the sub-steps after 2
    without a change; those groups are changed on fluid_floor_params."""
    c = CASES["fluid_clamp"]
    return _updated(c, {1: [(0, 1e3, c["models"][0]["vol"], (4e4, 7.15, 2.0))]}, [])


def _sand_floor_params():
    c = CASES["sand_floor"]
    v = c["models"][0]["vol"]
    return _updated(c, {56: [(0, 1e3, v, (2e4, 0.4))], 59: [(0, 1e3, v, (2e4, 0.25))]}, [])   # E, nu; ~100 particles on the yield branch


def _nacc_shear_params():
    c = CASES["nacc_shear"]
    v = c["models"][0]["vol"]
    ups = {}
    for k, args in ((4, (5e3, 0.4, 2.0, 0.8)), (7, (5e3, 0.4, 2.0, 0.3)), (10, (2e4, 0.4, 2.0, 0.3)), (13, (2e4, 0.25, 2.0, 0.3))):   # beta, xi, E, nu
        ups[k] = [(0, 1e3, v, args), (1, 1e3, v, args)]
    return _updated(c, ups, [])


def _multi_model_params():
    """multi_model_8 with rho changes to the second fixed-corotated model, the second fluid and the NACC model only: each update
    must reach its own slot of its material's g2p2g launch."""
    c = CASES["multi_model_8"]
    m = c["models"]
    return _updated(c, {1: [(1, 1e3, m[1]["vol"], m[1]["args"])],
                        2: [(4, 1.6e3, m[4]["vol"], m[4]["args"]), (6, 500.0, m[6]["vol"], m[6]["args"])]}, [0, 3])


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
    # particles on cell faces: exactly at (k + 1/2) dx and one ulp either side, below and above x = 0.5, at rest without
    # gravity and moving; a stencil's far corner then has weights of order 2^-39 per axis (64^3, below 0.5): its FP32 mass
    # is subnormal, and such a node holds no mass (quirk #9)
    "half_exact_lo": _half(6, 20, "exact"),
    "half_ulp_lo": _half(6, 20, "ulp"),
    "half_ulp_hi": _half(6, 36, "ulp"),
    "half_ulp_lo_moving": _half(6, 20, "ulp", v0=(0.3, -1.0, 0.2), gravity=-9.8),
    "half_ulp_db10_lo": _half(10, 300, "ulp"),
    "half_ulp_db10_hi": _half(10, 600, "ulp", v0=(0.3, -1.0, 0.2), gravity=-9.8),
    "half_ulp_top_corner": _half(6, 45, "ulp", v0=(0.5, 0.5, 0.5), gravity=-9.8),   # up to cell 63.5, stencils reach node 4G
    "half_ulp_lo_fluid": _half(6, 20, "ulp", v0=(0.3, -1.0, 0.2), gravity=-9.8, material=J_FLUID),
    # a cell overflow inside g2p2g: the layer's arrivals stay in their particle block (arrival lists of the sorted path) or
    # cross into the next one (phase 3)
    "overflow_fc_in_block": _overflow(FIXED_COROTATED, 27),
    "overflow_fluid_cross_block": _overflow(J_FLUID, 26),
    "nacc_soft_shear": _case(6, [model(NACC, box(1.0 / 64, (24, 20, 24), (36, 26, 36)), (2.0, -0.01, 0.0), 1.0 / 64, args=NACC_SOFT),
                                 model(NACC, box(1.0 / 64, (24, 26, 24), (36, 32, 36)), (-2.0, 0.01, 0.0), 1.0 / 64, args=NACC_SOFT)], [4, 7],
                             max_near_branch=0.25),
}
# parameter changes between sub-steps: odd and even update steps, each checked with the sub-step after it
CASES.update({
    "fc_floor_params": _fc_floor_params(),
    "fluid_floor_params": _fluid_floor_params(),
    "fluid_clamp_params": _fluid_clamp_params(),
    "sand_floor_params": _sand_floor_params(),
    "nacc_shear_params": _nacc_shear_params(),
    "multi_model_8_params": _multi_model_params(),
})


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


def kernel_level_inputs(ob, material, deform=False, steps=4, case=None):
    """The oracle after ``steps`` sub-steps of a small cube (or of ``case``), its grid turned into velocities by the oracle's
    grid update, and with deform=True the current bins' F replaced by extreme_f (the oracle's particle_state then reads them
    back)."""
    case = _cube(material, steps=[steps]) if case is None else case
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
    return Config(domain_bits=case["domain_bits"], max_ppc=case["max_ppc"], cfl=case["cfl"], gravity=case.get("gravity", -9.8),
                  boundary=case.get("boundary", 2))


def build_oracle(ob, case, max_blocks=6000):
    cfg = ob.make_config(domain_bits=case["domain_bits"], max_ppc=case["max_ppc"], cfl=case["cfl"], gravity=case.get("gravity", -9.8),
                         boundary=case.get("boundary", 2))
    if case.get("collider") or case.get("objects"):
        import collider_oracle_binding as cob
        sim = cob.ColliderOracleSim(cfg, case["dt"], max_blocks)
        if case.get("collider"):
            sdf, grad = collider_field(case)
            sim.set_collider(collider_struct(cob.Collider(), case["collider"]), sdf, grad)
        sim.set_collision_objects(object_structs(case))
    else:
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
    set_boundaries(sim, case)
    sim.initial_setup()
    return sim


def set_boundaries(sim, case):
    """The case's collider and collision objects on an engine simulator, before its initial_setup."""
    if case.get("collider"):
        sdf, grad = collider_field(case)
        p = collider_spec(case["collider"])
        sim.set_collider(sdf, grad, type=p["type"], friction=p["friction"], trans=p["trans"], trans_vel=p["trans_vel"], omega=p["omega"],
                         rot=np.asarray(p["rot_mat"]).reshape(3, 3), scale=p["scale"], dsdt=p["dsdt"])
    if case.get("objects"):
        sim.set_collision_objects(object_structs(case))


# ---- the collider of a case -------------------------------------------------------------------------------------------
def collider_spec(c):
    """A case's collider parameters with SignedDistanceGrid's defaults (identity rot_mat, no motion, scale 1)."""
    return dict(type=c["type"], friction=c.get("friction", 0.3), rot_mat=tuple(np.asarray(c.get("rot_mat", np.eye(3)), np.float64).reshape(9)),
                trans=tuple(c.get("trans", (0.0, 0.0, 0.0))), trans_vel=tuple(c.get("trans_vel", (0.0, 0.0, 0.0))),
                omega=tuple(c.get("omega", (0.0, 0.0, 0.0))), dsdt=c.get("dsdt", 0.0), scale=c.get("scale", 1.0))


def collider_struct(col, c):
    """Fill a cb200_collider / orc_collider ctypes struct (its sdf pointer left alone) from a case's collider."""
    p = collider_spec(c)
    col.rot_mat[:] = [float(v) for v in p["rot_mat"]]
    col.trans[:], col.trans_vel[:], col.omega[:] = [float(v) for v in p["trans"]], [float(v) for v in p["trans_vel"]], [float(v) for v in p["omega"]]
    col.dsdt, col.scale, col.friction, col.type = float(p["dsdt"]), float(p["scale"]), float(p["friction"]), int(p["type"])
    return col


_FIELDS = {}


def make_field(domain_bits, field, boundary=2):
    """(sdf (N, N, N), grad (3, N, N, N)) float32 of a field spec: ("box", lo, hi), ("sphere", centre, radius),
    ("plane", point, normal), ("zero_slab", y_top): sdf -1 at y <= y_top and +1 above, gradient 0 everywhere (quirk C5);
    ("solid",): sdf -1 and gradient (0, 1, 0) everywhere."""
    from claymore_b200 import levelset
    key = (domain_bits, repr(field))
    if key not in _FIELDS:
        cfg = Config(domain_bits=domain_bits, boundary=boundary)
        kind = field[0]
        N = 4 << (domain_bits - 2)
        if kind in ("box", "sphere", "plane"):
            out = getattr(levelset, kind)(cfg, *field[1:])
        elif kind == "zero_slab":
            y = np.arange(N) / float(1 << domain_bits)
            sdf = np.broadcast_to(np.where(y <= field[1], -1.0, 1.0)[None, :, None], (N, N, N)).astype(np.float32)
            out = (np.ascontiguousarray(sdf), np.zeros((3, N, N, N), np.float32))
        elif kind == "solid":
            grad = np.zeros((3, N, N, N), np.float32)
            grad[1] = 1.0
            out = (-np.ones((N, N, N), np.float32), grad)
        else:
            raise ValueError(kind)
        _FIELDS.clear()   # one field at a time: 4 MiB at 64^3, 256 MiB at 256^3
        _FIELDS[key] = out
    return _FIELDS[key]


def collider_field(case):
    return make_field(case["domain_bits"], case["collider"]["field"])


def ref_collider(case):
    """The (col, sdf, grad) argument of ref64.grid_update / substep for a case (None without a collider)."""
    if not case.get("collider"):
        return None
    sdf, grad = collider_field(case)
    return ref64.collider_params(collider_spec(case["collider"])), sdf, grad


STICKY, SLIP, SEPARATE = ref64.STICKY, ref64.SLIP, ref64.SEPARATE
FLOOR = ("box", (0.15, 0.15, 0.15), (0.85, 0.305, 0.85))   # a floor whose top (0.305) is not on a node (19.52 dx)


def _on_floor(material, typ, friction=0.3, steps=(0, 12, 30), **kw):
    """An 8 x 6 x 8-cell block falling at 6 m/s onto FLOOR: its stencils reach the floor's nodes (y <= 19 dx) at sub-step ~12."""
    dx = 1.0 / 64
    return _case(6, [model(material, box(dx, (26, 21, 26), (34, 27, 34)), (0.3, -6.0, 0.2), dx)], list(steps), dt=2e-4,
                 collider=dict(field=FLOOR, type=typ, friction=friction), **kw)


def _paddle(world_rot=(0.4, -0.3, 0.25), steps=(0, 3, 6)):
    """A box paddle through a resting fluid block with every motion at once: a non-identity rot_mat, trans, trans_vel, all three
    omega components, scale and dsdt; SLIP with friction 0.3.  The paddle moves at ~3 m/s, so the nodes it resolves set the max
    and dt is CFL-bound: cfl 0.05 keeps that dt (~2.5e-4) within the fluid's own stable step."""
    dx = 1.0 / 64
    return _case(6, [model(J_FLUID, box(dx, (18, 18, 18), (34, 34, 34)), (0.0, 0.0, 0.0), dx)], list(steps), dt=1e-3, cfl=0.05,
                 collider=dict(field=("box", (0.36, 0.30, 0.37), (0.43, 0.50, 0.44)), type=SLIP, friction=0.3, rot_mat=_rot(*world_rot),
                               trans=(0.40, 0.40, 0.40), trans_vel=(3.0, 0.5, -1.0), omega=(0.5, -0.7, 1.1), scale=1.1, dsdt=0.3))


def _thin_top():
    """boundary = 0: a block moving up into a sticky half-space y > 0.95 (nodes 61 .. 63); node 63 is solid, but its cell's
    +1 node (64 = 4G) does not exist, so the top guard (C6) leaves it alone."""
    dx = 1.0 / 64
    return _case(6, [model(FIXED_COROTATED, box(dx, (26, 57, 26), (34, 63, 34)), (0.2, 1.0, -0.1), dx)], [0, 2], boundary=0, gravity=0.0,
                 collider=dict(field=("plane", (0.5, 0.95, 0.5), (0.0, -1.0, 0.0)), type=STICKY, friction=0.0))


COLLIDER_CASES = {
    "floor_fc_sticky": _on_floor(FIXED_COROTATED, STICKY),
    "floor_fc_slip": _on_floor(FIXED_COROTATED, SLIP),
    "floor_fc_separate": _on_floor(FIXED_COROTATED, SEPARATE),
    "floor_fluid_slip": _on_floor(J_FLUID, SLIP),
    "floor_sand_sticky": dict(_on_floor(SAND, STICKY), max_near_branch=1.0),   # F = I at sub-step 0: the cone tip
    "floor_nacc_separate": _on_floor(NACC, SEPARATE),
    # frictionless SEPARATE on a sphere: normals in every direction
    "sphere_separate": _case(6, [model(FIXED_COROTATED, box(1.0 / 64, (26, 22, 26), (38, 28, 38)), (0.0, -2.0, 0.0), 1.0 / 64)], [0, 10],
                             collider=dict(field=("sphere", (0.5, 0.25, 0.5), 0.09), type=SEPARATE, friction=0.0)),
    "paddle_combined": _paddle(),
    # quirk C5: a slab of sdf -1 with a zero gradient; SLIP leaves the velocity as it is, SEPARATE stops it
    "zero_grad_slip": _case(6, [model(FIXED_COROTATED, box(1.0 / 64, (26, 18, 26), (34, 26, 34)), (0.3, -1.0, 0.2), 1.0 / 64)], [0, 3],
                            collider=dict(field=("zero_slab", 0.305), type=SLIP, friction=0.3)),
    "zero_grad_separate": _case(6, [model(FIXED_COROTATED, box(1.0 / 64, (26, 18, 26), (34, 26, 34)), (0.3, -1.0, 0.2), 1.0 / 64)], [0, 3],
                                collider=dict(field=("zero_slab", 0.305), type=SEPARATE, friction=0.3)),
    "thin_top_boundary0": _thin_top(),
    # quirk C1: a field that is solid everywhere; the wall-band nodes keep the update without the collider
    "walls_solid": dict(_walls(FIXED_COROTATED), collider=dict(field=("solid",), type=STICKY)),
    # a moving floor at the frame end: fps = 390 makes sub-step 25 end the frame with new_dt = 0.64 dt
    "moving_floor_frame_end": dict(_floor(FIXED_COROTATED, [24, 25, 26]), fps=390,
                                   collider=dict(field=("box", (0.15, 0.05, 0.15), (0.85, 0.2, 0.85)), type=SLIP, friction=0.3,
                                                 trans_vel=(0.2, 0.05, 0.0))),
    # the wall thickness without a collider.  boundary_bounds keeps them on the collider cases' bounds (ref64_checks): a wall
    # band's edge through walls_boundary1's models takes the oracle's F to 5.9 of KAPPA, under COLLIDER_KAPPA's 8
    "walls_boundary1": dict(_walls(FIXED_COROTATED, boundary=1), boundary_bounds=True),
    "fc_cube_boundary0": _cube(FIXED_COROTATED, steps=[0, 3], boundary=0, boundary_bounds=True),
}


# ---- analytic collision objects (DESIGN.md section 2.9) -------------------------------------------------------------------
# A case with ``objects`` = [(shape, args, keywords)] has analytic collision objects (claymore_b200.objects.<shape>(*args,
# **keywords)), resolved after its collider, if any, in list order (object_structs, ref_objects).
def make_object(shape, args, **kw):
    """claymore_b200.objects.<shape>(*args, **kw); shape "raw_plane" is a plane whose stored normal is the caller's as given,
    not of unit length: only cb200_sim_set_collision_objects' own normalisation makes it one."""
    from claymore_b200 import objects
    if shape != "raw_plane":
        return getattr(objects, shape)(*args, **kw)
    o = objects.plane(*args, **kw)
    o.b[:] = [float(v) for v in args[1]]
    return o


def object_structs(case):
    """The case's objects as cb200_collision_object structs (make_object)."""
    return [make_object(shape, args, **kw) for shape, args, kw in case.get("objects", ())]


def ref_objects(case):
    """The ``objects`` argument of ref64.grid_update / substep for a case (None without objects)."""
    return object_structs(case) or None


FLOOR_LO, FLOOR_HI = FLOOR[1], FLOOR[2]
# every motion at once, as _paddle's collider: a non-identity rot_mat, trans, trans_vel, all three omega components, scale, dsdt
PADDLE_MOTION = dict(rot=_rot(0.4, -0.3, 0.25), trans=(0.40, 0.40, 0.40), trans_vel=(3.0, 0.5, -1.0), omega=(0.5, -0.7, 1.1), scale=1.1, dsdt=0.3)


def _on_object_floor(material, typ, friction=0.3, steps=(12, 30), **kw):
    """_on_floor with FLOOR as an analytic box."""
    dx = 1.0 / 64
    return _case(6, [model(material, box(dx, (26, 21, 26), (34, 27, 34)), (0.3, -6.0, 0.2), dx)], list(steps), dt=2e-4,
                 objects=[("box", (FLOOR_LO, FLOOR_HI), dict(type=typ, friction=friction))], **kw)


def _falling(lo, hi, objs, steps=(10, 24), v0=(0.3, -6.0, 0.2), material=FIXED_COROTATED, dt=2e-4, **kw):
    """A block [lo, hi) (cells) falling onto the objects objs."""
    dx = 1.0 / 64
    return _case(6, [model(material, box(dx, lo, hi), v0, dx)], list(steps), dt=dt, objects=objs, **kw)


def _sixteen():
    """The longest list: five container planes around a fluid block and eleven small boxes and spheres inside the container,
    the last of them a sphere in the block's path."""
    objs = [("plane", ((0.5, 0.25, 0.5), (0.0, 1.0, 0.05)), dict(type=SLIP, friction=0.2)),
            ("plane", ((0.22, 0.5, 0.5), (1.0, 0.0, 0.0)), dict(type=SEPARATE, friction=0.0)),
            ("plane", ((0.62, 0.5, 0.5), (-1.0, 0.1, 0.0)), dict(type=SLIP, friction=0.0)),
            ("plane", ((0.5, 0.5, 0.22), (0.0, 0.0, 1.0)), dict(type=STICKY)),
            ("plane", ((0.5, 0.5, 0.62), (0.0, -0.05, -1.0)), dict(type=SEPARATE, friction=0.3))]
    for i in range(10):
        c = (0.27 + 0.033 * i, 0.3 + 0.011 * (i % 3), 0.27 + 0.031 * ((3 * i) % 10))
        if i % 2:
            objs.append(("sphere", (c, 0.017), dict(type=(SLIP, SEPARATE, STICKY)[i % 3], friction=0.3)))
        else:
            objs.append(("box", (tuple(x - 0.015 for x in c), tuple(x + 0.015 for x in c)), dict(type=(SLIP, SEPARATE, STICKY)[i % 3], friction=0.2)))
    objs.append(("sphere", ((0.47, 0.33, 0.46), 0.03), dict(type=SLIP, friction=0.3, trans_vel=(0.2, 0.0, 0.0))))
    return _falling((24, 20, 24), (36, 28, 36), objs, material=J_FLUID, v0=(0.2, -4.0, -0.1))


OBJECT_CASES = {
    "obj_floor_fc_sticky": _on_object_floor(FIXED_COROTATED, STICKY),
    "obj_floor_fc_slip": _on_object_floor(FIXED_COROTATED, SLIP),
    "obj_floor_fc_separate": _on_object_floor(FIXED_COROTATED, SEPARATE),
    "obj_floor_fluid_slip": _on_object_floor(J_FLUID, SLIP),
    "obj_floor_sand_sticky": dict(_on_object_floor(SAND, STICKY), max_near_branch=1.0),   # F = I at sub-step 0: the cone tip
    "obj_floor_nacc_separate": _on_object_floor(NACC, SEPARATE),
    # a tilted plane: a normal off every axis, passed without normalising it, and no lattice node within rounding of the plane
    "obj_tilted_plane_slip": _falling((24, 22, 24), (36, 28, 36), [("raw_plane", ((0.5, 0.3037, 0.5), (0.31, 1.0, -0.23)), dict(type=SLIP, friction=0.3))]),
    # frictionless SEPARATE on a sphere: normals in every direction
    "obj_sphere_separate": _falling((26, 22, 26), (38, 28, 38), [("sphere", ((0.5, 0.25, 0.5), 0.09), dict(type=SEPARATE, friction=0.0))],
                                    steps=(0, 10), v0=(0.0, -2.0, 0.0), dt=1e-4),
    # a capped cylinder tilted by rot_mat, under a block wider than it: the material meets the cap and the side
    "obj_cylinder_tilted": _falling((18, 23, 18), (46, 27, 46), [("cylinder", ((0.5, 0.26, 0.5), 0.1, 0.07), dict(type=SLIP, friction=0.3, rot=_rot(0.5, 0.3, 0.0), trans=(0.5, 0.26, 0.5)))],
                                    steps=(10, 20)),
    # static and lattice-aligned: faces at nodes 24 / 40 (x, z) and 16 / 24 (y), the centre at node (32, 20, 32); the nodes
    # equidistant from two faces and the centre are exact ties (E = 0), which the lowest axis and the + sign win.  A small
    # block rests at the centre, another falls onto the top face
    "obj_lattice_box": _case(6, [model(FIXED_COROTATED, box(1.0 / 64, (30, 18, 30), (34, 22, 34)), (0.0, 0.0, 0.0), 1.0 / 64),
                                 model(FIXED_COROTATED, box(1.0 / 64, (22, 25, 22), (42, 29, 42)), (0.0, -3.0, 0.0), 1.0 / 64)], [6, 12], dt=2e-4,
                             objects=[("box", ((0.375, 0.25, 0.375), (0.625, 0.375, 0.625)), dict(type=SLIP, friction=0.0))]),
    # static, centred on node (32, 16, 32), r = 8 dx, h = 12 dx: where d2 = 0 the nodes with |d1| = rho + 4 dx are exact cap / side
    # ties (E = 0), which the side wins (h - |d1| < r - rho is false); a block falls onto the cap and round its rim
    "obj_lattice_cylinder": _case(6, [model(FIXED_COROTATED, box(1.0 / 64, (22, 28, 22), (42, 32, 42)), (0.0, -3.0, 0.0), 1.0 / 64)], [0, 8], dt=2e-4,
                                  objects=[("cylinder", ((0.5, 0.25, 0.5), 0.125, 0.1875), dict(type=SLIP, friction=0.0))]),
    # the paddle with every motion at once through resting fluid: it sets the CFL-bound dt
    "obj_paddle_combined": _case(6, [model(J_FLUID, box(1.0 / 64, (18, 18, 18), (34, 34, 34)), (0.0, 0.0, 0.0), 1.0 / 64)], [0, 14], dt=1e-3, cfl=0.05,
                                 objects=[("box", ((0.36, 0.30, 0.37), (0.43, 0.50, 0.44)), dict(type=SLIP, friction=0.3, **PADDLE_MOTION))]),
    # overlapping objects: the list order decides where they overlap
    "obj_overlap": _falling((22, 24, 22), (42, 30, 42), [("sphere", ((0.5, 0.3, 0.5), 0.07), dict(type=STICKY, trans_vel=(0.1, 0.0, 0.0))),
                                                         ("box", ((0.4, 0.2, 0.4), (0.6, 0.33, 0.58)), dict(type=SLIP, friction=0.3)),
                                                         ("cylinder", ((0.45, 0.3, 0.52), 0.06, 0.08), dict(type=SEPARATE, friction=0.0, omega=(0.0, 0.7, 0.0)))]),
    # the level-set collider and two objects (the COLLIDE forms of the objects kernels)
    "obj_collider_plus_two": _falling((26, 22, 26), (38, 28, 38), [("box", (FLOOR_LO, (0.85, 0.2, 0.85)), dict(type=STICKY, trans_vel=(0.1, 0.0, 0.0))),
                                                                  ("sphere", ((0.56, 0.3, 0.45), 0.05), dict(type=SEPARATE, friction=0.3))],
                                      collider=dict(field=("sphere", (0.45, 0.25, 0.5), 0.09), type=SLIP, friction=0.3, trans_vel=(0.2, 0.0, 0.0))),
    "obj_sixteen": _sixteen(),
    # objects have no wall-band guard: a slip box through the floor band (cells y < 8) under a column standing in it, and at
    # boundary 0 a sticky box over the top faces, where node 63 = 4G - 1 has mass
    "obj_wall_band": dict(_floor(FIXED_COROTATED, [0, 10]), objects=[("box", ((0.1, -0.1, 0.1), (0.9, 0.2, 0.9)), dict(type=SLIP, friction=0.3, trans_vel=(0.2, 0.0, 0.0)))]),
    "obj_top_boundary0": _case(6, [model(FIXED_COROTATED, box(1.0 / 64, (26, 57, 26), (34, 63, 34)), (0.2, 1.0, -0.1), 1.0 / 64)], [0, 2], boundary=0,
                               gravity=0.0, objects=[("box", ((0.0, 0.95, 0.0), (1.0, 1.1, 1.0)), dict(type=STICKY))]),
    # a moving floor at the frame end: fps = 390 makes sub-step 25 end the frame with new_dt = 0.64 dt
    "obj_moving_floor_frame_end": dict(_floor(FIXED_COROTATED, [24, 25, 26]), fps=390,
                                       objects=[("box", ((0.15, 0.05, 0.15), (0.85, 0.2, 0.85)), dict(type=SLIP, friction=0.3, trans_vel=(0.2, 0.05, 0.0)))]),
}
