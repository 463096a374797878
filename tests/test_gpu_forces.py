"""The boundary impulse report (DESIGN.md section 2.13) on the GPU.

Kernel level: cb200_update_grid_velocity_query_max_forces over the analytic-object matrix of test_ref64_objects_cpu against
ref64_forces.boundary_impulses per body within its derived bound, the grid bit-identical to the entry without the report and the
max within MAX_ULPS, and the balance identity.  Step driver: 40 sub-steps of static, moving and turning bodies, the level-set
collider and level-set objects, every sub-step against the reference on the grid it read (the level-set instances also on vs off
on those grids); two MGSP ranks whose partials sum to the whole; a sand column's weight and torque on a floor; resets, rejections
and the scene runner's --forces file and its resume.
"""
import ctypes as C

import numpy as np
import pytest

import ref64
import ref64_cases as S
import ref64_forces as RF
import ref64_levelset as RL
from ref64_checks import build_ranks, on_threads, rank_grid
from test_levelset_objects_cpu import level_set
from test_ref64_collider_cpu import FIELDS, MOTIONS, TIMES, block_field
from test_ref64_mgsp_cpu import split_case
from test_ref64_objects_cpu import ENTRIES, entry_runs, kernel_config, synthetic_grid

pytestmark = pytest.mark.gpu

EPS32 = 2.0 ** -24
FLOOR_LS = level_set("box")
DRAGON_LS = level_set("dragonish")


@pytest.fixture(scope="module")
def force_kernel(cuda_lib):
    """run(cfg, keys, grid, dt, collider spec or None, objects, t, report) -> (grid, max, impulses[1 + n, 6] or None)"""
    import torch
    from claymore_b200 import objects
    from claymore_b200._capi import Collider, Config, Partition
    cfg0 = Config(domain_bits=6)
    sdf, grad = S.make_field(cfg0.domain_bits, FIELDS["sphere"])
    field = torch.from_numpy(block_field(cfg0.domain_bits, sdf, grad)).cuda()

    def run(cfg, keys, grid, dt, spec, objs, t, report=True, impulses=None):
        col = None
        if spec is not None:
            col = S.collider_struct(Collider(), spec)
            col.sdf = field.data_ptr()
        g = torch.from_numpy(np.ascontiguousarray(grid)).cuda()
        k = torch.from_numpy(np.ascontiguousarray(keys.reshape(-1))).cuda()
        mv = torch.zeros(1, dtype=torch.float32, device="cuda")
        part = Partition()
        part.active_keys = k.data_ptr()
        ecfg = Config(domain_bits=cfg.domain_bits, boundary=cfg.boundary, gravity=cfg.gravity)
        common = (C.byref(ecfg), len(keys), C.c_void_p(g.data_ptr()), part, dt, C.byref(col) if col is not None else None, objects.array(objs), len(objs),
                  None, 0, float(np.float32(t)), C.c_void_p(mv.data_ptr()))
        imp = None
        if report:
            imp = impulses if impulses is not None else torch.zeros((1 + len(objs)) * 6, dtype=torch.float64, device="cuda")
            assert cuda_lib.cb200_update_grid_velocity_query_max_forces(*common, C.c_void_p(imp.data_ptr()), None) == 0
        else:
            assert cuda_lib.cb200_update_grid_velocity_query_max_levelsets(*common, None) == 0
        torch.cuda.synchronize()
        return g.cpu().numpy(), float(mv.item()), (imp.cpu().numpy().reshape(-1, 6) if imp is not None else None)
    return run


def _ref_collider(cfg, spec):
    if spec is None:
        return None
    sdf, grad = S.make_field(cfg.domain_bits, FIELDS["sphere"])
    return ref64.collider_params(spec), sdf, grad


def _balance(cfg, keys, grid, dt, post, imp):
    """(sum over bodies of J, the float64 momentum the chain removed from the GPU's own velocities, its FP32 bound)"""
    has, m, v0, _ = RF.pre_chain_velocity(cfg, keys.astype(np.int64), grid, dt)
    vout = post[:, 1:].astype(np.float64)
    dj = np.where(has[:, None], m[:, None] * (v0 - vout), 0.0)
    want = dj.sum((0, 2))
    # v0 recomputed in float64: its FP32 rounding (|v| 2^-24 per product and the gravity add) and the kernel's FP32 sums
    bound = 4 * EPS32 * (np.where(has[:, None], m[:, None] * np.abs(v0), 0.0).sum((0, 2)) + RF.SUM_ULPS * np.abs(dj).sum((0, 2)))
    return imp[:, :3].sum(0), want, bound


MATRIX = [(e, b, m) for e in ENTRIES for b in (2, 0) for m in MOTIONS]
MAX_ULPS = 4.0   # |max_on - max_off| / (2^-24 max_off): a sum of three squares rounded in two orders
VEL_KAPPA = 2 * RF.VEL_KAPPA   # both instances lie within VEL_KAPPA 2^-24 E of ref64 per node (E: ref64's error magnitude)


def _same_velocities(cfg, keys, grid, dt, ccol, t, objs, post, post0, label):
    """The reporting level-set-object instance without the collider is compiled into other multiply-adds than the one without the
    report (DESIGN.md section 2.13): the masses bit for bit, and every velocity within the kernel bound of the other, both being
    within ref64's (nodes ref64 flags near a discontinuity left out, as the kernel tests do).  Returns (values that differ, worst
    |v_on - v_off| / (2^-24 E))."""
    assert np.array_equal(post[:, 0].view(np.uint32), post0[:, 0].view(np.uint32)), f"{label}: masses differ"
    _, mag, _, info = ref64.grid_update(cfg, keys, grid, dt, ccol, np.float32(t), objs)
    d = np.abs(post[:, 1:].astype(np.float64) - post0[:, 1:].astype(np.float64))
    keep = ~info["near"][:, None, :]
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(keep & (d > 0), d / (EPS32 * mag), 0.0)
    assert np.nan_to_num(ratio, nan=np.inf).max(initial=0.0) <= VEL_KAPPA, f"{label}: velocities {ratio.max()} x 2^-24 E apart"
    return int((post.view(np.uint32) != post0.view(np.uint32)).sum()), float(ratio.max(initial=0.0))


@pytest.mark.parametrize("entry,boundary,motion", MATRIX, ids=[f"{e}-b{b}-{m}" for e, b, m in MATRIX])
def test_kernel_impulses_match_ref64(oracle, force_kernel, entry, boundary, motion):
    cfg = kernel_config(oracle, boundary)
    dt = 1e-4
    worst, loaded, worst_max = 0.0, 0, 0.0
    for ti, t in enumerate(TIMES):
        for ri, (rl, spec, objs) in enumerate(entry_runs(entry, motion)):
            if ri % 3 == 0:
                keys, grid = synthetic_grid(cfg, objs, spec, t, seed=ti + 10 * boundary + 100 * ENTRIES.index(entry))
            label = f"{entry} b{boundary} {motion} {rl} t {t}"
            post, mx, imp = force_kernel(cfg, keys, grid, dt, spec, objs, t)
            # report on vs off: the same velocities bit for bit; the max |v|^2 of those same velocities may round differently (DESIGN.md
            # section 2.13: the two instances sum the three squares in another FP32 order), within MAX_ULPS
            post0, mx0, _ = force_kernel(cfg, keys, grid, dt, spec, objs, t, report=False)
            assert np.array_equal(post.view(np.uint32), post0.view(np.uint32)), f"{label}: the reporting grid update resolved other velocities"
            assert abs(mx - mx0) <= MAX_ULPS * EPS32 * mx0, f"{label}: max {mx} vs {mx0}"
            worst_max = max(worst_max, abs(mx - mx0) / (EPS32 * mx0) if mx0 > 0 else 0.0)
            r = RF.boundary_impulses(cfg, keys.astype(np.int64), grid, dt, _ref_collider(cfg, spec), t, objs)
            for name, got, want, bound in (("J", imp[:, :3], r["J"], r["bJ"]), ("L", imp[:, 3:], r["L"], r["bL"])):
                err = np.abs(got - want)
                assert (err <= bound).all(), f"{label}: {name} {got} vs ref64 {want}, bound {bound}"
                worst = max(worst, float(np.max(np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), 0.0))))
            if spec is None:
                assert not imp[0].any(), f"{label}: no collider, but body 0 reports {imp[0]}"
            loaded += int((np.abs(imp[:, :3]).sum(1) > 0).sum())
            got, want, bound = _balance(cfg, keys, grid, dt, post, imp)
            assert (np.abs(got - want) <= bound).all(), f"{label}: sum of J {got} vs removed momentum {want}, bound {bound}"
    assert loaded > 0
    print(f"{entry} b{boundary} {motion}: worst {worst:.3f} of the derived bound, {loaded} loaded bodies, max |v|^2 off by {worst_max:.2f} x 2^-24")


def test_kernel_no_hit_is_zero_and_calls_accumulate(oracle, force_kernel):
    import torch
    from claymore_b200 import objects
    cfg = kernel_config(oracle, 2)
    keys, grid = synthetic_grid(cfg, [objects.sphere((0.5, 0.5, 0.5), 0.21)], None, 0.0, seed=7)
    far = [objects.sphere((0.05, 0.05, 0.05), 0.01, type="sticky")]            # in the wall band's corner: no block there
    _, _, imp = force_kernel(cfg, keys, grid, 1e-4, None, far, 0.0)
    assert not imp.any(), imp
    objs = [objects.box((0.3, 0.28, 0.33), (0.68, 0.61, 0.7), type="slip", friction=0.3)]
    _, _, once = force_kernel(cfg, keys, grid, 1e-4, None, objs, 0.37)
    acc = torch.zeros(12, dtype=torch.float64, device="cuda")
    force_kernel(cfg, keys, grid, 1e-4, None, objs, 0.37, impulses=acc)
    _, _, twice = force_kernel(cfg, keys, grid, 1e-4, None, objs, 0.37, impulses=acc)
    assert np.abs(once[1]).sum() > 0
    assert np.allclose(twice, 2 * once, rtol=1e-12, atol=0.0)


# ---- step driver ----------------------------------------------------------------------------------------------------------
DX = 1.0 / 64
FLOOR_TOP = 0.3


def _column(sim_kw, lo, hi, ppc_side=2):
    """(sim, particle mass total): a sand block at rest, 8 particles per cell, standing on a sticky floor box whose top is FLOOR_TOP
    (sand piles up and comes to rest; a fluid would spread to the walls)"""
    from claymore_b200 import GmpmSimulator, objects
    from claymore_b200._capi import Config
    sim = GmpmSimulator(config=Config(domain_bits=6), max_blocks=4000, dt=2e-4, **sim_kw)
    h = DX / ppc_side
    axes = [np.arange(lo[d] + h / 2, hi[d], h) for d in range(3)]
    pos = np.stack(np.meshgrid(*axes, indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
    mid = sim.init_model(S.SAND, pos)
    rho, vol = 1000.0, (h ** 3)
    sim.update_sand_parameters(rho, vol, 1e5, 0.3, model=mid)
    sim.set_collision_objects([objects.box((0.1, 0.13, 0.1), (0.9, FLOOR_TOP, 0.9), type="sticky", trans=(0.5, 0.2, 0.5))])
    mass = len(pos) * float(np.float32(np.float32(rho) * np.float32(vol)))
    return sim, mass


@pytest.mark.timeout(900)
@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
def test_column_weight_and_torque_on_floor(cuda_lib, use_graph):
    """A sand column settled on a floor box: the mean vertical force over the last frames is the column's weight (mass x gravity,
    downward), and the torque about the box's pivot (0.5, 0.2, 0.5) is -d W about z for a column off it by d along x."""
    d = 0.125
    sim, mass = _column(dict(fps=48, frames=40, use_graph=use_graph), (0.5 + d - 0.0625, FLOOR_TOP, 0.4375), (0.5 + d + 0.0625, FLOOR_TOP + 0.125, 0.5625))
    try:
        sim.initial_setup()
        sim.report_forces()
        W = -9.8 * mass
        F, T = [], []
        for f in range(1, 41):
            sim.advance_frame()
            el, imp = sim.collision_forces()
            assert el > 0
            F.append(imp[1, :3] / el)
            T.append(imp[1, 3:] / el)
        assert sim.stats().error == 0
        F, T = np.array(F[-10:]), np.array(T[-10:])
        print(f"graph={use_graph}: Fy/W over the last 10 frames {F[:, 1].min() / W:.5f} .. {F[:, 1].max() / W:.5f}; "
              f"Tz/(d W) {T[:, 2].min() / (d * W):.5f} .. {T[:, 2].max() / (d * W):.5f}; |Fx|, |Fz| <= {np.abs(F[:, [0, 2]]).max() / abs(W):.2e} W")
        assert np.abs(F[:, 1].mean() / W - 1) < 0.02
        assert np.abs(T[:, 2].mean() / (d * W) - 1) < 0.03
        assert np.abs(F[:, [0, 2]].mean(0)).max() < 0.02 * abs(W)
    finally:
        sim.close()


@pytest.mark.timeout(900)
def test_centred_column_has_no_torque(cuda_lib):
    sim, mass = _column(dict(fps=48, frames=30), (0.4375, FLOOR_TOP, 0.4375), (0.5625, FLOOR_TOP + 0.125, 0.5625))
    try:
        sim.initial_setup()
        sim.report_forces()
        for f in range(25):
            sim.advance_frame()
            sim.collision_forces()
        sim.advance_frame()
        el, imp = sim.collision_forces()
        W = 9.8 * mass
        print(f"centred: Fy/W {-imp[1, 1] / el / W:.5f}, |T| / (W dx) {np.abs(imp[1, 3:]).max() / el / (W * DX):.2e}")
        assert np.abs(imp[1, 3:]).max() / el < 0.01 * W * DX
    finally:
        sim.close()


def test_accumulator_resets_and_spans_sim_time(cuda_lib):
    from claymore_b200 import CB200Error, objects
    sim, _ = _column(dict(fps=48, frames=4), (0.4375, FLOOR_TOP, 0.4375), (0.5625, FLOOR_TOP + 0.0625, 0.5625))
    try:
        sim.initial_setup()
        with pytest.raises(CB200Error):
            sim.collision_forces()                                           # the report is off
        sim.report_forces()
        t0 = sim.sim_time()
        sim.step(5)
        el, imp = sim.collision_forces()
        assert el == sim.sim_time() - t0 and imp.shape == (2, 6) and imp[1, 1] < 0
        t1 = sim.sim_time()
        sim.step(3)
        sim.set_collision_objects([objects.box((0.1, 0.13, 0.1), (0.9, FLOOR_TOP, 0.9), type="slip"),
                                   objects.sphere((0.2, 0.8, 0.2), 0.05)])   # resets: the rows change meaning
        t2 = sim.sim_time()
        assert t2 > t1
        el, imp = sim.collision_forces()
        assert el == 0.0 and imp.shape == (3, 6) and not imp.any()
        sim.step(4)
        el, imp = sim.collision_forces()
        assert el == sim.sim_time() - t2 and imp[1, 1] < 0 and not imp[2].any()
        sim.report_forces(False)
        with pytest.raises(CB200Error):
            sim.collision_forces()
    finally:
        sim.close()


@pytest.mark.timeout(900)
def test_scene_forces_file_and_resume(cuda_lib, tmp_path):
    """python -m claymore_b200 --forces: one row per frame and body, the column's weight on the floor; a run resumed from frame 2's
    checkpoint appends rows for frames 3.. that match the uninterrupted run's within the parity bounds"""
    import json

    import claymore_b200.__main__ as M
    from claymore_b200 import scene
    doc = {"simulation": {"default_dt": 2e-4, "fps": 48, "frames": 5},
           "models": [{"constitutive": "sand", "type": "particles", "file": "box", "offset": [0.4375, 0.3125, 0.4375],
                       "span": [0.125, 0.0625, 0.125], "rho": 1000, "volume": (DX / 2) ** 3, "youngs_modulus": 1e5, "poisson_ratio": 0.3}],
           "boundaries": [{"shape": "box", "offset": [0.1, 0.13, 0.1], "span": [0.8, FLOOR_TOP - 0.13, 0.8], "type": "sticky"},
                          {"shape": "sphere", "offset": [0.15, 0.8, 0.15], "span": [0.05, 0.05, 0.05]}]}
    path = tmp_path / "s.json"
    path.write_text(json.dumps(doc))
    full, part = tmp_path / "full", tmp_path / "part"
    full.mkdir()
    part.mkdir()
    assert M.main(["-f", str(path), "--out", str(full), "--forces"]) == 0
    rows = [r.split(",") for r in (full / "forces.csv").read_text().strip().split("\n")]
    assert rows[0] == list(scene.FORCE_COLUMNS) and len(rows) == 1 + 5 * 3
    assert [r[3] for r in rows[1:4]] == ["none", "box", "sphere"]
    box = [float(r[5]) for r in rows[1:] if r[3] == "box"]
    rest = [float(x) for r in rows[1:] if r[3] != "box" for x in r[4:]]
    assert box[-1] < 0 and not any(rest), f"box Fy per frame {box}, other bodies {rest}"
    # the same run through the API, stopping at frame 2 for a checkpoint
    sim = scene.parse_scene(str(path), forces=True)
    ck = str(tmp_path / "f2.ckpt")
    on_frame, fh = scene.force_recorder(sim, str(part / "forces.csv"))
    try:
        sim.initial_setup()
        for f in (1, 2):
            sim.advance_frame()
            on_frame(sim, f)
        sim.save_checkpoint(ck)
    finally:
        fh.close()
        sim.close()
    assert M.main(["-f", str(path), "--out", str(part), "--forces", "--resume", ck]) == 0
    prow = [r.split(",") for r in (part / "forces.csv").read_text().strip().split("\n")]
    assert [r[:4] for r in prow] == [r[:4] for r in rows]
    a = np.array([[float(x) for x in r[4:]] for r in rows[1:]])
    b = np.array([[float(x) for x in r[4:]] for r in prow[1:]])
    # g2p2g's atomic sums make the two runs' grids differ in the last bits, and the frames after the checkpoint follow them
    assert np.allclose(a, b, rtol=1e-2, atol=1e-2 * np.abs(a).max())


# ---- the step driver, sub-step by sub-step, against the float64 reference -------------------------------------------------
def _union(sims):
    """(keys, grid) of the ranks' grids, each block once: the lowest rank's copy (a halo block's reduced sums are on every holder),
    and the keys held by more than one rank"""
    parts = [rank_grid(s) for s in sims]
    keys = np.concatenate([k for k, _ in parts])
    grid = np.concatenate([g for _, g in parts])
    uk, first, cnt = np.unique(keys, axis=0, return_index=True, return_counts=True)
    return keys[first], grid[first], uk[cnt > 1]


def driver_force_check(sims, case, steps, label, kernel=None):
    """Each of `steps` sub-steps: the grid every rank's update reads and the clock, then one sub-step, then the rows the ranks
    report, summed, against ref64_forces.boundary_impulses on that grid at that t and dt, within its bound; the span each rank
    reports is the sub-step's dt.  kernel(keys, grid, dt, t) (single domain): kernel-level checks on the same grid.  Returns the
    largest |J| the reference puts on blocks more than one rank holds (0 for one rank)."""
    cfg = sims[0].cfg
    ccol, objs = S.ref_collider(case), S.object_structs(case) if case.get("objects") else []
    for s in sims:
        s.report_forces()
    halo, loaded = 0.0, 0
    for k in range(steps):
        st = [s.stats() for s in sims]
        dt, t = st[0].dt, sims[0].sim_time()
        assert all(x.dt == dt for x in st) and all(s.sim_time() == t for s in sims), f"{label}: ranks disagree on the clock"
        keys, grid, shared = _union(sims)
        if kernel is not None:
            kernel(keys, grid, dt, t)
        r = RF.boundary_impulses(cfg, keys, grid, dt, ccol, np.float32(t), objs)
        if len(shared):
            m = (keys[:, None, :] == shared[None]).all(-1).any(1)
            h = RF.boundary_impulses(cfg, keys[m], grid[m], dt, ccol, np.float32(t), objs)
            halo = max(halo, float(np.abs(h["J"]).max()))
        if len(sims) > 1:
            on_threads(sims, lambda s: s.step(1))
        else:
            sims[0].step(1)
        assert all(s.stats().error == 0 for s in sims), f"{label}: error bits at sub-step {k}"
        got = np.zeros_like(np.concatenate([r["J"], r["L"]], 1))
        for s in sims:
            el, imp = s.collision_forces()
            assert el == s.sim_time() - t, f"{label}: span {el} for a sub-step from {t}"
            got += imp
        for name, g, want, bound in (("J", got[:, :3], r["J"], r["bJ"]), ("L", got[:, 3:], r["L"], r["bL"])):
            assert (np.abs(g - want) <= bound).all(), f"{label} sub-step {k}: {name} {g} vs ref64 {want}, bound {bound}"
        loaded += int((np.abs(got[:, :3]).sum(1) > 0).sum())
    assert loaded > 0, f"{label}: no body was ever loaded"
    return halo


LS_FLOOR = ("levelset", (FLOOR_LS, (0.2, -0.336, 0.2117), (0.61, 0.88, 0.5333)))
DRIVER_CASES = {
    "floor_sticky": S.OBJECT_CASES["obj_floor_fc_sticky"],
    "floor_slip": S.OBJECT_CASES["obj_floor_fc_slip"],
    "floor_separate": S.OBJECT_CASES["obj_floor_fc_separate"],
    "collider_plus_two": S.OBJECT_CASES["obj_collider_plus_two"],
    "paddle_combined": S.OBJECT_CASES["obj_paddle_combined"],
    # level-set objects (the grid update's LEVELSETS instances): a floor, the moving, turning dragon, and a level set after the
    # dense collider and between two analytic objects
    "levelset_floor": S._case(6, [S.model(S.FIXED_COROTATED, S.box(DX, (26, 24, 26), (34, 30, 34)), (0.3, -3.0, 0.2), DX)], [], dt=2e-4,
                              objects=[LS_FLOOR + (dict(type=S.SLIP, friction=0.3),)]),
    "levelset_dragon": S._case(6, [S.model(S.J_FLUID, S.box(DX, (26, 32, 24), (36, 40, 40)), (0.0, -2.0, 0.0), DX)], [], dt=2e-4,
                               objects=[("levelset", (DRAGON_LS, (0.42, 0.42, 0.25), (0.5, 0.5, 0.5)),
                                         dict(type=S.SLIP, friction=0.2, trans=(0.47, 0.49, 0.5), trans_vel=(0.0, 0.3, 0.1), omega=(0.2, 1.5, -0.4),
                                              scale=1.05, dsdt=0.1))]),
    "levelset_with_collider": S._case(6, [S.model(S.FIXED_COROTATED, S.box(DX, (26, 28, 26), (38, 34, 36)), (0.3, -3.0, 0.2), DX)], [], dt=2e-4,
                                      collider=dict(type=S.SLIP, friction=0.0, field=("plane", (0.5, 0.2, 0.5), (0.2, 1.0, 0.0))),
                                      objects=[("box", ((0.4, 0.36, 0.4), (0.47, 0.42, 0.6)), dict(type=S.SLIP, friction=0.3)),
                                               LS_FLOOR + (dict(type=S.SEPARATE, friction=0.3),), ("sphere", ((0.56, 0.38, 0.5), 0.05), dict(type=S.STICKY))]),
}


def _lattices(case):
    seen = [args[0] for shape, args, _ in case.get("objects", ()) if shape == "levelset"]
    assert all(s is seen[0] for s in seen), "ref64_cases' structs carry index 0: one level set per case"
    return [RL.lattice(ls.n, ls.phi) for ls in seen[:1]]


def _levelset_kernel(cuda_lib, case, lats):
    """kernel(keys, grid, dt, t): the reporting kernel entry with the case's level-set objects against the one without the report
    (the same velocities bit for bit, the max within MAX_ULPS) and the balance identity, on the driver's own grid"""
    import torch
    from claymore_b200 import objects
    from claymore_b200._capi import Collider, LevelSetLattice, Partition
    dev = [torch.from_numpy(np.ascontiguousarray(l)).cuda() for l in lats]
    lv = (LevelSetLattice * len(dev))(*[LevelSetLattice(d.data_ptr(), l.shape[2], l.shape[1], l.shape[0]) for d, l in zip(dev, lats)])
    field = None
    if case.get("collider"):
        sdf, grad = S.collider_field(case)
        field = torch.from_numpy(block_field(case["domain_bits"], sdf, grad)).cuda()
    objs = S.object_structs(case)
    cfg = S.config(case)

    def run(keys, grid, dt, t):
        col = None
        if field is not None:
            col = S.collider_struct(Collider(), S.collider_spec(case["collider"]))
            col.sdf = field.data_ptr()
        outs = []
        for report in (True, False):
            g = torch.from_numpy(np.ascontiguousarray(grid)).cuda()
            k = torch.from_numpy(np.ascontiguousarray(keys.astype(np.int32).reshape(-1))).cuda()
            mv = torch.zeros(1, dtype=torch.float32, device="cuda")
            imp = torch.zeros((1 + len(objs)) * 6, dtype=torch.float64, device="cuda")
            part = Partition()
            part.active_keys = k.data_ptr()
            common = (C.byref(cfg), len(keys), C.c_void_p(g.data_ptr()), part, dt, C.byref(col) if col is not None else None, objects.array(objs), len(objs),
                      lv, len(dev), float(np.float32(t)), C.c_void_p(mv.data_ptr()))
            if report:
                assert cuda_lib.cb200_update_grid_velocity_query_max_forces(*common, C.c_void_p(imp.data_ptr()), None) == 0
            else:
                assert cuda_lib.cb200_update_grid_velocity_query_max_levelsets(*common, None) == 0
            torch.cuda.synchronize()
            outs.append((g.cpu().numpy(), float(mv.item()), imp.cpu().numpy().reshape(-1, 6)))
        (post, mx, imp), (post0, mx0, _) = outs
        n, worst = _same_velocities(cfg, keys, grid, dt, S.ref_collider(case), t, objs, post, post0, "level-set objects")
        DIFFS.append((n, post.size, worst))
        assert abs(mx - mx0) <= MAX_ULPS * EPS32 * mx0, f"max {mx} vs {mx0}"
        got, want, bound = _balance(cfg, keys, grid, dt, post, imp)
        assert (np.abs(got - want) <= bound).all(), f"sum of J {got} vs removed momentum {want}, bound {bound}"
    return run


DIFFS = []


@pytest.mark.timeout(900)
@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
@pytest.mark.parametrize("name", list(DRIVER_CASES))
def test_driver_impulses_match_ref64(cuda_lib, name, use_graph):
    """40 sub-steps of the step driver, every one against the float64 reference on the grid it read, the bodies placed at the
    engine's sim_time: static, moving and turning bodies, the level-set collider and level-set objects"""
    case = DRIVER_CASES[name]
    lats = _lattices(case)
    with RL.registered(lats):
        sim = S.build_engine(case, use_graph=use_graph)
        try:
            DIFFS.clear()
            driver_force_check([sim], case, 40, f"{name} {'graph' if use_graph else 'stream'}", _levelset_kernel(cuda_lib, case, lats) if lats else None)
        finally:
            sim.close()
    if DIFFS:
        print(f"{name}: report on vs off, {sum(d[0] for d in DIFFS)} of {sum(d[1] for d in DIFFS)} grid values differ, worst "
              f"{max(d[2] for d in DIFFS):.2f} x 2^-24 E")


@pytest.mark.timeout(900)
@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
def test_mgsp_partials_sum_to_the_whole(cuda_lib, use_graph):
    """Two x slabs of a block falling onto a sticky floor box that the halo between them crosses: the ranks' rows, summed, match
    the reference on the union of their grids (each block once), sub-step by sub-step.  A halo block counted on both ranks would
    add the halo's share twice; the test requires that share to be loaded."""
    case = S._case(6, [S.model(S.FIXED_COROTATED, S.box(DX, (24, 20, 24), (36, 28, 34)), (1.0, -10.0, 0.5), DX)], [], dt=1e-3,
                   objects=[("box", (S.FLOOR_LO, S.FLOOR_HI), dict(type=S.STICKY, friction=0.3))])
    sims = build_ranks(case, split_case(case, 2, "x"), use_graph)
    try:
        halo = driver_force_check(sims, case, 30, f"MGSP 2x {'graph' if use_graph else 'stream'}")
    finally:
        for s in sims:
            s.close()
    assert halo > 0, "no halo block was loaded: the test could not see a halo counted twice"


def test_collision_forces_validation_changes_nothing(cuda_lib):
    """Every rejection of cb200_sim_collision_forces leaves the sums and their span as they were; adding particles keeps them."""
    from claymore_b200 import objects
    sim, _ = _column(dict(fps=48, frames=4), (0.4375, FLOOR_TOP, 0.4375), (0.5625, FLOOR_TOP + 0.0625, 0.5625))
    try:
        sim.set_collision_objects([objects.box((0.1, 0.13, 0.1), (0.9, FLOOR_TOP, 0.9), type="sticky"), objects.sphere((0.2, 0.8, 0.2), 0.05)])
        sim.initial_setup()
        sim.report_forces()
        t0 = sim.sim_time()
        sim.step(5)
        out = np.zeros((17, 6), np.float64)
        n, el = C.c_int(-7), C.c_double(-7.0)
        L, h, p = sim.L, sim.h, C.c_void_p(out.ctypes.data)
        assert L.cb200_sim_collision_forces(h, None, 17, C.byref(n), C.byref(el)) != 0
        assert L.cb200_sim_collision_forces(h, p, 17, None, C.byref(el)) != 0
        assert L.cb200_sim_collision_forces(h, p, 17, C.byref(n), None) != 0
        assert L.cb200_sim_collision_forces(h, p, 2, C.byref(n), C.byref(el)) != 0      # 3 rows
        assert (n.value, el.value) == (-7, -7.0) and not out.any()
        sim.add_particles(0, np.array([[0.5, 0.6, 0.5], [0.51, 0.6, 0.5]], np.float32))
        sim.step(2)
        assert L.cb200_sim_collision_forces(h, p, 3, C.byref(n), C.byref(el)) == 0
        assert n.value == 3 and el.value == sim.sim_time() - t0 and out[1, 1] < 0
    finally:
        sim.close()
