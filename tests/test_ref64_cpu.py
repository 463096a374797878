"""The float64 reference (tests/ref64.py) against the FP32 oracle, one sub-step at a time, and its own identities.

For every case: the oracle's state at sub-step k -> ref64 for one sub-step -> compared with the oracle at k + 1 per grid
cell (by key) and per particle (matched by position), each against its own bound kappa * 2^-24 * M (ref64.compare).
The kappa values below are the smallest round values the FP32 oracle passes over this whole matrix; the GPU tests
(test_gpu_ref64.py) hold the engine to the same values.
"""
import numpy as np
import pytest

import ref64
import ref64_cases as S

# kappa per quantity; beside each, the oracle's worst |oracle - ref64| / (2^-24 M) over CASES
KAPPA = dict(
    mass=1.0,       # oracle worst 0.63 (domain_bits_5)
    momentum=0.2,   # oracle worst 0.127 (fluid_clamp); M includes the sensitivity to the stored position's last bit
    pos=2.0,        # oracle worst 1.89 (fluid_clamp)
    F=4.0,          # oracle worst 3.4 (cfl_bound; J, F, logJp)
)
# set-up rasterisation sums up to 27 x 8 terms per node in any order, and its M has no position-sensitivity term
RASTER_KAPPA = dict(mass=32.0, momentum=32.0, pos=1.0, F=1.0)   # oracle worst 19.4 (walls)
# a constitutive model's own error, in units of its stress scale (DESIGN.md section 3, device math unit tests):
# fixed-corotated 3e-5 of (2 mu + lambda) vol |F|^2; sand and NACC 3e-5 of the stress, 2e-5 of F and logJp
STRESS_ALLOW = 3e-5
F_ALLOW = {ref64.J_FLUID: 0.0, ref64.FIXED_COROTATED: 0.0, ref64.SAND: 2e-5, ref64.NACC: 2e-5}
BRANCH_MARGIN = 1e-4
# The new dt is sqrt, then a division, after the max of FP32 |v|^2: three roundings, so one ulp (what a single correctly
# rounded operation would give) is not reachable in FP32.  The oracle's worst case is 1.01 ulp (cfl_bound); 2 is the next
# whole number of ulps.
DT_ULPS = 2.0
# grid update (kernel level): v = mv * (1 / m), masked, + g dt: a few roundings of the magnitude |mv / m| + |g dt|
VEL_KAPPA = 4.0   # oracle worst 2.13; the max |v|^2 within 4 x 2^-24 relative (oracle worst 1.63)


def check_report(rep, label):
    for q in ("mass", "momentum", "pos", "F"):
        assert rep[q] <= 1.0, f"{label}: {q} error is {rep[q]:.3g} x its bound ({rep['worst']})"


def check_dt(impl_dt, ref_dt, label):
    ulp = float(np.spacing(np.float32(ref_dt)))
    assert abs(impl_dt - ref_dt) <= DT_ULPS * ulp, f"{label}: dt {impl_dt!r} vs reference {ref_dt!r} ({(impl_dt - ref_dt) / ulp:.2f} ulp)"


def ref_models(case, states):
    return [dict(material=m["material"], params=S.ref_params(m), state=s) for m, s in zip(case["models"], states)]


def oracle_substep_check(ob, case, label):
    """Run the oracle through case['steps']; at each, one ref64 sub-step against the oracle's next one."""
    osim = S.build_oracle(ob, case)
    clock = S.OracleClock(osim)
    nm = len(case["models"])
    done = 0
    near = 0
    worst = dict(mass=0.0, momentum=0.0, pos=0.0, F=0.0)
    for k in case["steps"]:
        clock.step(k - done)
        _, nbc, _ = osim.block_counts()
        r = ref64.substep(osim.cfg, ref_models(case, [osim.particle_state(i) for i in range(nm)]), osim.active_keys()[:nbc], osim.grid(),
                          osim.dt, case["dt"], clock.time_left())
        clock.step(1)
        done = k + 1
        _, nbc, _ = osim.block_counts()
        rep = ref64.compare(r, osim.active_keys()[:nbc], osim.grid(), [osim.particle_state(i) for i in range(nm)], KAPPA,
                            STRESS_ALLOW, [F_ALLOW[m["material"]] for m in case["models"]], margin=BRANCH_MARGIN)
        check_report(rep, f"{label} sub-step {k}")
        check_dt(osim.dt, r["new_dt"], f"{label} sub-step {k}")
        near += rep["near_branch"]
        for q in worst:
            worst[q] = max(worst[q], rep[q])
    osim.close()
    return worst, near


@pytest.mark.parametrize("name", [n for n, c in S.CASES.items() if c.get("oracle", True)])
def test_ref64_matches_oracle(oracle, name):
    case = S.CASES[name]
    worst, near = oracle_substep_check(oracle, case, name)
    total = sum(len(m["pos"]) for m in case["models"]) * len(case["steps"])
    # the branch-point exclusion is for the odd particle; a case where it hides a large share proves nothing
    assert near <= case.get("max_near_branch", 0.01) * total, f"{name}: {near} of {total} particle updates within {BRANCH_MARGIN} of a branch point"


@pytest.mark.parametrize("cases,want", [(("sand_floor",), {"tip", "elastic", "yield"}),
                                         (("nacc_floor", "nacc_shear"), {"elastic", "expand", "compress", "project_harden"})],
                         ids=["sand", "nacc"])
def test_ref64_sand_and_nacc_take_every_branch(oracle, cases, want):
    """The plastic cases reach the return-mapping branches their bounds are stated for, with particles away from the branch
    points; the branch is the one ref64 takes from each particle's trial state.  (NACC's projection without a hardening
    update needs p0 <= 1e-4 or a trial pressure within 1e-4 of the cap, which no case reaches.)"""
    got = set()
    for name in cases:
        case = S.CASES[name]
        nm = len(case["models"])
        for k in case["steps"]:
            osim = S.build_oracle(oracle, case)
            osim.step(k)
            _, nbc, _ = osim.block_counts()
            r = ref64.substep(osim.cfg, ref_models(case, [osim.particle_state(i) for i in range(nm)]), osim.active_keys()[:nbc], osim.grid(),
                              osim.dt, case["dt"])
            for res in r["models"]:
                got |= set(np.unique(res["branch"][res["margin"] >= BRANCH_MARGIN]).tolist())
            osim.close()
    assert want <= got, (cases, got)


# ---- kernel level: the oracle's drop-in kernels on identical containers ---------------------------------------------------
KERNEL_LEVEL = [(S.FIXED_COROTATED, True), (S.FIXED_COROTATED, False), (S.J_FLUID, False), (S.NACC, False)]
# At det F ~ 0.1, inverted or nearly singular F the stress comes from a 4-sweep Jacobi SVD: the reference's own (the oracle's)
# and the device's fall-back of the same scheme.  That SVD is up to 6e-4 of the stress scale away from the exact one on such
# F (DESIGN.md section 3, device math unit tests), so those particles get 3e-5 + 1.5 x 6e-4, about 1e-3, instead of 3e-5.
SVD_STRESS_ALLOW = 1e-3


def check_grid_update(cfg, keys, pre, post, mx_impl, dt, label):
    """An implementation's grid update (post, mx_impl) of the grid ``pre`` against ref64.grid_update."""
    vel, vmag, mx = ref64.grid_update(cfg, keys, pre, dt)
    post = np.asarray(post, np.float64)
    assert np.array_equal(post[:, 0], pre[:, 0]), f"{label}: the grid update changed the mass channel"
    err = np.abs(post[:, 1:] - vel)
    bound = VEL_KAPPA * ref64.EPS32 * vmag
    assert np.all(err <= bound), f"{label}: grid velocity error {np.max(err / np.maximum(bound, 1e-300)):.3g} x its bound"
    assert abs(mx_impl - mx) <= 4 * ref64.EPS32 * mx, f"{label}: max |v|^2 {mx_impl!r} vs {mx!r}"
    return vel


def kernel_level_check(ob, material, deform, run_grid_update, run_g2p2g, label):
    """Containers from the oracle (S.kernel_level_inputs); ``run_grid_update(g0) -> (grid, max)`` and ``run_g2p2g(velocity grid)
    -> (next grid, next bins)`` are the implementation under test, both on copies of the oracle's containers."""
    case, osim = S.kernel_level_inputs(ob, material, deform)
    pbc, nbc, _ = osim.block_counts()
    cfg, dt = osim.cfg, osim.dt
    keys = osim.partition_arrays(0)["active_keys"].reshape(-1, 3)[:nbc].astype(np.int64)
    pre = osim.grid_array(0)[: nbc * 256].reshape(nbc, 4, 64).astype(np.float64)
    post, mx = run_grid_update(osim)
    check_grid_update(cfg, keys, pre, post.reshape(nbc, 4, 64), mx, dt, label)
    # g2p2g from the oracle's FP32 velocities (the kernel's input), at the state its bins hold (deformed F included)
    vel32 = osim.grid_array(0)[: nbc * 256].reshape(nbc, 4, 64)[:, 1:].astype(np.float64)
    states = [osim.particle_state(0)]
    r = ref64.g2p2g(cfg, ref_models(case, states), keys, vel32, np.abs(vel32), dt, dt)
    g1, bins = run_g2p2g(osim)
    nxt = osim.buffer_arrays(0, 1)
    se = S.states_from_bins(bins, nxt["bin_offsets"], nxt["particle_bucket_sizes"], pbc, material)
    allow = SVD_STRESS_ALLOW if deform else STRESS_ALLOW
    rep = ref64.compare(r, keys, g1.reshape(-1, 4, 64)[:nbc], [se], KAPPA, allow, [F_ALLOW[material]], margin=BRANCH_MARGIN)
    check_report(rep, label)
    osim.close()
    return rep


def oracle_grid_update(ob):
    def run(osim):
        import ctypes as C
        _, nbc, _ = osim.block_counts()
        mv = np.zeros(1, np.float32)
        g0 = osim.grid_array(0)
        ob.lib().orc_update_grid_velocity_query_max(C.byref(osim.cfg), nbc, ob.ptr(g0), osim.partition_arrays(0)["struct"], osim.dt, ob.ptr(mv))
        return g0[: nbc * 256].copy(), float(mv[0])
    return run


def oracle_g2p2g(ob):
    def run(osim):
        import ctypes as C
        pbc, nbc, ebc = osim.block_counts()
        cur, nxt = osim.buffer_arrays(0, 0), osim.buffer_arrays(0, 1)
        g1 = osim.grid_array(1)
        g1[: nbc * 256] = 0
        nxt["cell_particle_counts"][: ebc * 64] = 0
        ob.lib().orc_g2p2g(C.byref(osim.cfg), osim.dt, osim.dt, pbc, cur["struct"], nxt["struct"], osim.partition_arrays(1)["struct"],
                           osim.partition_arrays(0)["struct"], ob.ptr(osim.grid_array(0)), ob.ptr(g1))
        return g1[: nbc * 256].copy(), nxt["bins"].copy()
    return run


@pytest.mark.parametrize("material,deform", KERNEL_LEVEL)
def test_ref64_matches_oracle_kernel_level(oracle, material, deform):
    """orc_update_grid_velocity_query_max and orc_g2p2g on the containers the GPU kernel-level test feeds cb200_*; with
    deform=True the particles carry F at det ~ 0.1, inverted, nearly singular and stretched (S.extreme_f)."""
    kernel_level_check(oracle, material, deform, oracle_grid_update(oracle), oracle_g2p2g(oracle), f"oracle kernel level {material} {deform}")


# ---- identities of the reference itself ----------------------------------------------------------------------------------
def test_bspline_partition_of_unity_and_zero_first_moment():
    rng = np.random.default_rng(1)
    dx_inv = 64.0
    pos = np.concatenate([rng.uniform(0.1, 0.9, (2000, 3)), (np.arange(20, 40)[:, None] + np.array([0.5, 0.0, -0.5 + 1e-12])) / dx_inv])
    base, d, W, G, xixp, off = ref64.stencil(pos, dx_inv)
    assert np.all((d >= 0.5 - 1e-12) & (d <= 1.5 + 1e-12))
    assert np.abs(W.sum(1) - 1).max() <= 1e-14
    assert np.abs(np.einsum("nk,nkd->nd", W, xixp)).max() <= 1e-14 / dx_inv
    # second moment of the quadratic B-spline: sum w (x_i - x_p)^2 = dx^2 / 4 per axis (APIC's D = dx^2 / 4 I)
    assert np.abs(np.einsum("nk,nkd->nd", W, xixp ** 2) - 0.25 / dx_inv ** 2).max() <= 1e-14 / dx_inv ** 2
    # round half away from zero at cell faces
    assert list(ref64.cell_index(np.array([0.5, 1.5, 2.5, 2.4999999]) / dx_inv, dx_inv)) == [1, 2, 3, 2]


def test_apic_transfer_conserves_linear_and_angular_momentum():
    """G2P -> P2G with zero stress, no gravity and no walls: total momentum and angular momentum (particles' affine part
    included) are conserved to 1e-12 relative."""
    from claymore_b200._capi import Config
    rng = np.random.default_rng(7)
    cfg = Config(domain_bits=6, boundary=0, gravity=0.0)
    dx = 1.0 / 64
    pos = rng.uniform(20 * dx, 40 * dx, (3000, 3))
    p = ref64.params(ref64.J_FLUID, 1e3, dx ** 3 / 8, 0.0, 7.15, 0.0)   # bulk 0, viscosity 0: no stress
    # a grid velocity field: rotation + shear + noise on the nodes around the particles
    keys = np.stack(np.meshgrid(*[np.arange(3, 12)] * 3, indexing="ij"), -1).reshape(-1, 3)
    cells = np.stack(np.meshgrid(np.arange(4), np.arange(4), np.arange(4), indexing="ij"), -1).reshape(64, 3)
    xn = (keys[:, None, :] * 4 + cells[None]) * dx - 0.5
    vel = np.stack([-xn[..., 1] + 0.3 * xn[..., 2], xn[..., 0], 0.2 * xn[..., 0]], 1) + 0.01 * rng.standard_normal((len(keys), 3, 64))
    st = np.concatenate([pos, np.ones((len(pos), 1))], 1)
    r = ref64.g2p2g(cfg, [dict(material=ref64.J_FLUID, params=p, state=st)], keys, vel, np.abs(vel), 0.0, 0.0)
    res = r["models"][0]
    m = p["mass"]
    # particle side: momentum m v, angular momentum x x m v + the affine part m (D^-1 sum w v (x_i - x_p))... expressed via C
    v = res["v"]
    base, d, W, G, xixp, off = ref64.stencil(pos, 64.0)
    nv, _ = ref64.Grid(keys, vel).gather(base[:, None, :] + off[None])
    A = np.einsum("nk,nkc,nkd->ncd", W, nv, xixp)
    C = A * 4 * 64 * 64                                                 # C = A D^-1
    P_p = m * v.sum(0)
    L_p = m * np.cross(pos, v).sum(0) + m * (0.25 / 64 ** 2) * np.stack([C[:, 2, 1] - C[:, 1, 2], C[:, 0, 2] - C[:, 2, 0], C[:, 1, 0] - C[:, 0, 1]], -1).sum(0)
    g = r["grid"]
    nodes = (r["keys"][:, None, :] * 4 + cells[None]) * dx
    mom = g[:, 1:].transpose(0, 2, 1)
    P_g = mom.sum((0, 1))
    L_g = np.cross(nodes, mom).sum((0, 1))
    assert np.abs(g[:, 0].sum() - m * len(pos)) <= 1e-12 * m * len(pos)
    assert np.abs(P_g - P_p).max() <= 1e-12 * np.abs(P_p).max()
    assert np.abs(L_g - L_p).max() <= 1e-12 * np.abs(L_p).max()


def test_rasterize_matches_oracle_setup(oracle):
    """Set-up rasterisation: the oracle's grid right after initial_setup against ref64.rasterize."""
    for name in ("walls", "multi_model_8"):
        case = S.CASES[name]
        osim = S.build_oracle(oracle, case)
        _, nbc, _ = osim.block_counts()
        keys, grid, mag = ref64.rasterize(osim.cfg, [dict(pos=m["pos"], v0=m["v0"], mass=S.ref_params(m)["mass"]) for m in case["models"]])
        r = dict(keys=keys, grid=grid, mag=mag, stress=np.zeros_like(grid), models=[])
        rep = ref64.compare(r, osim.active_keys()[:nbc], osim.grid(), [], RASTER_KAPPA, 0.0, [])
        check_report(rep, f"{name} rasterize")
        osim.close()


def test_wall_mask_on_both_faces_then_gravity():
    """ref64.grid_update: the mask on every low and high band, then gravity (quirk #1), NaN -> +inf (quirk #3)."""
    from claymore_b200._capi import Config
    cfg = Config(domain_bits=6, boundary=2, gravity=-9.8)
    G = 16
    keys = np.array([[1, 8, 8], [2, 8, 8], [13, 8, 8], [14, 8, 8], [8, 1, 8], [8, 14, 8], [8, 13, 8], [8, 8, 0], [8, 8, 15], [8, 8, 8]])
    grid = np.zeros((len(keys), 4, 64))
    grid[:, 0] = 2.0
    grid[:, 1:] = 2.0 * np.array([1.0, 2.0, 3.0])[None, :, None]
    v, _, mx = ref64.grid_update(cfg, keys, grid, 1e-3)
    gdt = float(np.float32(-9.8)) * 1e-3
    for k, vv in zip(keys, v):
        wall = (k < 2) | (k >= G - 2)
        want = np.where(wall, 0.0, [1.0, 2.0, 3.0]) + np.array([0, gdt, 0])
        assert np.allclose(vv, want[:, None], rtol=0, atol=1e-15), (k, vv[:, 0])
    grid[0, 1, 5] = np.nan
    keys[0] = (8, 8, 8)
    assert ref64.grid_update(cfg, keys, grid, 1e-3)[2] == np.inf
