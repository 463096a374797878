"""GPU tests of removing particles from a set-up simulator (cb200_sim_remove_particles / _remove_rows, GmpmSimulator.remove_particles /
remove_rows, the scene's "sinks").

The survivors are exactly the rows not selected, bitwise; the partition is the one a set-up over the survivors builds; grid[0] holds
the survivors' rasterisation at the velocities every node had before (DESIGN.md section 2.10), so each survivor's velocity is kept and
the next sub-step matches ref64.  Every rejection and every no-op leaves a checkpoint byte-identical to the one before it.
"""
import json
import os

import numpy as np
import pytest

import ref64
import ref64_cases as S
from claymore_b200 import bgeo, checkpoint, objects
from claymore_b200._capi import CB200Error, Config
from claymore_b200.scene import parse_scene, sink_schedule
from claymore_b200.simulator import GmpmSimulator
from ref64_checks import BRANCH_MARGIN, F_ALLOW, KAPPA, RASTER_KAPPA, STRESS_ALLOW, check_counts, check_dt, check_report, ref_models
from test_gpu_checkpoint import _assert_round_trip, _restored, _sorted_rows
from test_gpu_emit import _assert_same_classes
from test_gpu_parity import _compare_state

pytestmark = pytest.mark.gpu

DX = 1.0 / 64
MATERIALS = [S.FIXED_COROTATED, S.J_FLUID, S.SAND, S.NACC]
EPS = 2.0 ** -24
ULPS = 4


def _odd_cube(material, v0=(0.3, -1.0, 0.2)):
    """11^3 cells x 8 = 10648 particles: not a multiple of the compaction's 2048-row tile"""
    return S._case(6, [S.model(material, S.box(DX, (20, 20, 20), (31, 31, 31)), v0, DX)], [])


def _expected_removed(regions, pos, t, outside):
    """(removed[n], near[n]) of the union of the regions by the float64 reference; `near` rows lie within ref64's rounding
    margin of a surface"""
    hit = np.zeros(len(pos), bool)
    near = np.zeros(len(pos), bool)
    for o in regions:
        p = ref64.object_params(o)
        q = ref64.object_query(p, ref64.material_point(None, p, t, points=pos)["x"])
        hit |= q["hit"]
        near |= q["margin"] <= ref64.NEAR
    return (~hit if outside else hit), near


def _rows_after(before, removed):
    return _sorted_rows(before[~removed])


MOVING = dict(trans_vel=(0.4, -0.3, 0.2), omega=(0.0, 2.0, 1.0), dsdt=0.5)


def _regions(kind, moving):
    c = np.array([26.3, 25.7, 26.1]) * DX
    m = MOVING if moving else {}
    if kind == "box":
        return [objects.box(c - 3.1 * DX, c + 2.9 * DX, **m)]
    if kind == "sphere":
        return [objects.sphere(c, 4.2 * DX, **m)]
    if kind == "cylinder":
        return [objects.cylinder(c, 3.3 * DX, 4.4 * DX, **m)]
    return [objects.plane(c, (0.3, 1.0, -0.2), **m)]


@pytest.mark.parametrize("outside", [False, True], ids=["inside", "outside"])
@pytest.mark.parametrize("moving", [False, True], ids=["static", "moving"])
@pytest.mark.parametrize("kind", ["box", "sphere", "cylinder", "plane"])
@pytest.mark.parametrize("material", MATERIALS)
def test_region_rows(cuda_lib, material, kind, moving, outside):
    sim = S.build_engine(_odd_cube(material))
    sim.step(6)
    t = sim.sim_time()
    assert t > 0
    before = sim.particle_state(0)
    regions = _regions(kind, moving)
    removed, near = _expected_removed(regions, before[:, :3], np.float32(t), outside)
    got = sim.remove_particles(regions, outside=outside)
    after = sim.particle_state(0)
    assert got == [len(before) - len(after)] and sim.counts[0] == len(after)
    # every survivor is a row of before, bitwise; away from the surfaces the selection is the float64 reference's
    keep_sure, gone_sure = ~removed & ~near, removed & ~near
    a = {r.tobytes() for r in after}
    b = [r.tobytes() for r in before]
    assert a <= set(b)
    assert all(b[i] in a for i in np.flatnonzero(keep_sure)), "a row away from every surface was removed"
    assert not any(b[i] in a for i in np.flatnonzero(gone_sure)), "a row away from every surface survived"
    assert 0 < len(after) < len(before)
    sim.step(3)
    assert sim.stats().error == 0
    sim.close()


@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
@pytest.mark.parametrize("outside", [False, True], ids=["inside", "outside"])
def test_lattice_aligned_box_and_planes_are_exact(cuda_lib, use_graph, outside):
    """At t = 0 a lattice-aligned box and axis planes select exactly the float32 set (object_query on the stored float)."""
    sim = S.build_engine(_odd_cube(S.FIXED_COROTATED, v0=(0.0, 0.0, 0.0)), use_graph=use_graph)
    before = sim.particle_state(0)
    p = before[:, :3]
    lo, hi = np.float32(np.array([22.0, 21.0, 23.0]) * DX), np.float32(np.array([27.0, 26.0, 30.0]) * DX)
    regions = [objects.box(lo, hi), objects.plane((0.0, np.float32(29.0 * DX), 0.0), (0.0, -1.0, 0.0))]
    inside = np.all((p >= lo) & (p <= hi), 1) | (p[:, 1] >= np.float32(29.0 * DX))
    removed = ~inside if outside else inside
    assert sim.remove_particles(regions, outside=outside) == [int(removed.sum())]
    assert _sorted_rows(sim.particle_state(0)).tobytes() == _rows_after(before, removed).tobytes()
    sim.close()


def test_remove_rows_equals_boolean_indexing(cuda_lib):
    case = S._case(6, [S.model(S.J_FLUID, S.box(DX, (14, 20, 20), (25, 31, 31)), (0.5, -0.5, 0.0), DX),
                       S.model(S.NACC, S.box(DX, (30, 22, 20), (41, 33, 31)), (0.0, -0.8, 0.2), DX)], [])
    sim = S.build_engine(case)
    sim.step(5)
    rng = np.random.default_rng(3)
    for model in (1, 0):
        before = sim.particle_state(model)
        mask = rng.random(len(before)) < 0.37
        other = sim.particle_state(1 - model)
        assert sim.remove_rows(model, mask)[model] == mask.sum()
        assert _sorted_rows(sim.particle_state(model)).tobytes() == _sorted_rows(before[~mask]).tobytes()
        assert sim.particle_state(1 - model).tobytes() == other.tobytes() or \
            _sorted_rows(sim.particle_state(1 - model)).tobytes() == _sorted_rows(other).tobytes()
    sim.step(5)
    assert sim.stats().error == 0
    sim.close()


@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
def test_mid_run_removal_state(cuda_lib, tmp_path, use_graph):
    """Partition, grid, invariants and the clock after a removal from two models mid-run, and the sub-step after it."""
    case = S._case(6, [S.model(S.J_FLUID, S.box(DX, (14, 20, 20), (25, 31, 31)), (0.5, -0.5, 0.0), DX),
                       S.model(S.SAND, S.box(DX, (27, 22, 20), (38, 33, 31)), (0.0, -0.8, 0.2), DX)], [])
    sim = S.build_engine(case, use_graph=use_graph)
    sim.step(10)
    a = checkpoint.read(sim.save_checkpoint())
    d0 = str(tmp_path / "before")
    os.mkdir(d0)
    sim.write_frame(d0, 1, attributes=("v",))
    sim.wait_output()
    lo, hi = np.array([20.0, 24.0, 18.0]) * DX, np.array([31.0, 27.5, 33.0]) * DX
    region = [objects.box(lo, hi)]
    removed = sim.remove_particles(region)
    assert all(n > 0 for n in removed)
    b = checkpoint.read(sim.save_checkpoint())
    # the clock, bitwise
    for f in ("dt", "next_dt", "steps", "sim_time", "step_time", "frame_time", "frames", "error"):
        assert a[f] == b[f], f
    # survivors bitwise; partition = a set-up over them
    for m in range(2):
        pa = a["states"][m][:, :3]
        gone = np.all((pa >= np.float32(lo)) & (pa <= np.float32(hi)), 1)
        assert gone.sum() == removed[m]
        assert _sorted_rows(b["states"][m]).tobytes() == _rows_after(a["states"][m], gone).tobytes()
    fresh = S.build_engine(S._case(6, [dict(m, pos=b["states"][i][:, :3].copy()) for i, m in enumerate(case["models"])], []))
    _assert_same_classes(sim, fresh, "removal vs a set-up on the survivors")
    fresh.close()
    # grid: mass = rasterisation of the survivors; p/m kept at every node with m' > 0; no block beyond the new partition
    survivors = [dict(pos=b["states"][m][:, :3], v0=(0.0, 0.0, 0.0), mass=S.ref_params(cm)["mass"]) for m, cm in enumerate(case["models"])]
    rk, rg, rmag = ref64.rasterize(sim.cfg, survivors)
    old = {tuple(k): g for k, g in zip(a["keys"], a["grid"])}
    ref = {tuple(k): (g, mg) for k, g, mg in zip(rk, rg, rmag)}
    assert len(b["keys"]) == sim.stats().neighbor_block_count
    for k, g in zip(b["keys"], b["grid"].astype(np.float64)):
        k = tuple(k)
        assert k in old, "a block the state before did not have"
        rgk, mgk = ref.get(k, (np.zeros((4, 64)), np.zeros((4, 64))))
        assert (np.abs(g[0] - rgk[0]) <= RASTER_KAPPA["mass"] * EPS * mgk[0] + 1e-30).all(), "mass"
        o = old[k].astype(np.float64)
        live = g[0] > 0
        assert (o[0][live] > 0).all()
        v_new, v_old = g[1:, live] / g[0, live], o[1:, live] / o[0, live]
        assert (np.abs(v_new - v_old) <= ULPS * EPS * np.abs(v_old) + 1e-30).all(), "node velocity"
        assert (g[1:, ~live] == 0).all()
    # total mass and momentum drop by the removed particles' mass and (frame-output) momentum
    d1 = str(tmp_path / "after")
    os.mkdir(d1)
    sim.write_frame(d1, 1, attributes=("v",))
    sim.wait_output()
    ga, gb = a["grid"].astype(np.float64), b["grid"].astype(np.float64)
    for m, cm in enumerate(case["models"]):
        fa = bgeo.read(os.path.join(d0, f"model_id[{m}]_frame[1].bgeo"))
        fb = bgeo.read(os.path.join(d1, f"model_id[{m}]_frame[1].bgeo"))
        va = {r.tobytes(): v for r, v in zip(fa["position"], fa["v"])}
        for r, v in zip(fb["position"], fb["v"]):
            w = va.pop(r.tobytes())
            assert (np.abs(v.astype(np.float64) - w) <= ULPS * EPS * np.abs(w).max() + 1e-30).all(), "survivor velocity"
        assert len(va) == removed[m]
    mp = [S.ref_params(cm)["mass"] for cm in case["models"]]
    dm = sum(n * m for n, m in zip(removed, mp))
    assert abs((ga[:, 0].sum() - gb[:, 0].sum()) - dm) <= 1e-5 * ga[:, 0].sum()
    gone_p = np.zeros(3)
    for m in range(2):
        fa = bgeo.read(os.path.join(d0, f"model_id[{m}]_frame[1].bgeo"))
        keep = {r.tobytes() for r in b["states"][m][:, :3]}
        sel = np.array([r.tobytes() not in keep for r in fa["position"]])
        gone_p += mp[m] * fa["v"][sel].astype(np.float64).sum(0)
    for d in range(3):
        assert abs((ga[:, 1 + d].sum() - gb[:, 1 + d].sum()) - gone_p[d]) <= 1e-5 * np.abs(ga[:, 1 + d]).sum() + 1e-12
    # one sub-step against ref64, then 20 more equal to a restore of the state after the removal
    st = sim.stats()
    g = sim.grid()
    keys, before = sim.active_keys()[: len(g)], [sim.particle_state(i) for i in range(2)]
    r = ref64.substep(sim.cfg, ref_models(case, before), keys, g, st.dt, case["dt"])
    sim.step(1)
    assert sim.stats().error == 0
    g = sim.grid()
    states = [sim.particle_state(i) for i in range(2)]
    check_counts(r, before, states, case["max_ppc"], "sub-step after the removal")
    rep = ref64.compare(r, sim.active_keys()[: len(g)], g, states, KAPPA, STRESS_ALLOW, [F_ALLOW[m["material"]] for m in case["models"]],
                        margin=BRANCH_MARGIN, max_ppc=case["max_ppc"])
    check_report(rep, "sub-step after the removal")
    check_dt(sim.stats().dt, r["new_dt"], "sub-step after the removal")
    blob = sim.save_checkpoint()
    rs = _restored(blob, use_graph=use_graph)
    _assert_round_trip(sim, rs, 2)
    sim.step(20)
    rs.step(20)
    _compare_state(rs, sim, 2, "20 sub-steps after a removal", pos_tol=5e-6, f_tol=2e-4)
    rs.close()
    sim.close()


def test_empty_model(cuda_lib, tmp_path):
    """Emptying one of two models: the other steps as the reference says, frames hold 0 points, checkpoints are refused with the
    simulator unchanged, and add_particles refills the model."""
    far = S.model(S.FIXED_COROTATED, S.box(DX, (14, 20, 20), (22, 28, 28)), (0.2, -0.5, 0.0), DX)
    other = S.model(S.J_FLUID, S.box(DX, (38, 20, 36), (46, 28, 44)), (0.0, -0.5, 0.0), DX)
    case = S._case(6, [far, other], [])
    sim = S.build_engine(case)
    sim.step(3)
    n1 = len(sim.particle_state(1))
    assert sim.remove_rows(1, np.ones(n1, bool)) == [0, n1]
    assert sim.counts[1] == 0 and len(sim.particle_state(1)) == 0 and len(sim.retrieve(1)) == 0
    one = S._case(6, [far], [])
    for i in range(20):
        st = sim.stats()
        g = sim.grid()
        keys, before = sim.active_keys()[: len(g)], [sim.particle_state(0)]
        r = ref64.substep(sim.cfg, ref_models(one, before), keys, g, st.dt, case["dt"])
        sim.step(1)
        assert sim.stats().error == 0
        g = sim.grid()
        states = [sim.particle_state(0)]
        rep = ref64.compare(r, sim.active_keys()[: len(g)], g, states, KAPPA, STRESS_ALLOW, [F_ALLOW[far["material"]]], margin=BRANCH_MARGIN,
                            max_ppc=case["max_ppc"])
        check_report(rep, f"sub-step {i} with an empty model")
        assert len(sim.particle_state(1)) == 0
    paths = sim.write_frame(str(tmp_path), 1)
    sim.wait_output()
    assert len(bgeo.read(paths[1])["position"]) == 0 and len(bgeo.read(paths[0])["position"]) == len(sim.particle_state(0))
    state = sim.particle_state(0).tobytes()
    with pytest.raises(CB200Error, match="CUDA error 801 "):
        sim.checkpoint_begin()
    assert sim.particle_state(0).tobytes() == state
    with pytest.raises(CB200Error, match="CUDA error 1 "):   # the whole simulator would be empty
        sim.remove_rows(0, np.ones(len(sim.particle_state(0)), bool))
    add = S.box(DX, (38, 30, 36), (42, 34, 40))
    assert sim.add_particles(1, add, (0.0, -1.0, 0.0)) == len(add)
    blob = sim.save_checkpoint()
    rs = _restored(blob)
    _assert_round_trip(sim, rs, 2)
    sim.step(5)
    rs.step(5)
    _compare_state(rs, sim, 2, "5 sub-steps after a refill", pos_tol=5e-6, f_tol=2e-4)
    rs.close()
    sim.close()


def test_rejections_and_no_ops_leave_the_simulator_unchanged(cuda_lib):
    case = _odd_cube(S.FIXED_COROTATED)
    pos = case["models"][0]["pos"]
    fresh = GmpmSimulator(dt=1e-4, fps=0, config=S.config(case), max_blocks=4000)
    fresh.init_model(S.FIXED_COROTATED, pos, (0, 0, 0))
    with pytest.raises(CB200Error, match="CUDA error 1 "):       # not set up
        fresh.remove_particles([objects.sphere((0.4, 0.4, 0.4), 0.05)])
    fresh.close()
    sim = S.build_engine(case)
    sim.step(4)
    before = sim.save_checkpoint()
    n = len(sim.particle_state(0))
    box = objects.box((0.3, 0.3, 0.3), (0.4, 0.4, 0.4))
    arr = objects.array([box])
    bad = objects.box((0.3, 0.3, 0.3), (0.4, 0.4, 0.4))
    bad.a[0] = 0.5   # lo > hi
    L, h = sim.L, sim.h
    raw = {
        "empty mask": lambda: L.cb200_sim_remove_particles(h, 0, arr, 1, 0, None),
        "unknown model bit": lambda: L.cb200_sim_remove_particles(h, 2, arr, 1, 0, None),
        "unknown flags": lambda: L.cb200_sim_remove_particles(h, 1, arr, 1, 2, None),
        "invalid region": lambda: L.cb200_sim_remove_particles(h, 1, (objects.CollisionObject * 1)(bad), 1, 0, None),
        "n < 0": lambda: L.cb200_sim_remove_particles(h, 1, arr, -1, 0, None),
        "n > 16": lambda: L.cb200_sim_remove_particles(h, 1, (objects.CollisionObject * 17)(*([box] * 17)), 17, 0, None),
        "unknown model": lambda: L.cb200_sim_remove_rows(h, 1, np.zeros(n, np.uint8).ctypes.data_as(type(h)), n, None),
        "short mask": lambda: L.cb200_sim_remove_rows(h, 0, np.zeros(n, np.uint8).ctypes.data_as(type(h)), n - 1, None),
        "long mask": lambda: L.cb200_sim_remove_rows(h, 0, np.zeros(n + 1, np.uint8).ctypes.data_as(type(h)), n + 1, None),
        "everything": lambda: L.cb200_sim_remove_rows(h, 0, np.ones(n, np.uint8).ctypes.data_as(type(h)), n, None),
        "everything outside nothing": lambda: L.cb200_sim_remove_particles(h, 1, objects.array([objects.sphere((0.9, 0.9, 0.9), 0.01)]), 1, 1, None),
    }
    for name, fn in raw.items():
        assert fn() == 1, name
        assert sim.save_checkpoint().tobytes() == before.tobytes(), name
    with pytest.raises(ValueError):
        sim.remove_particles([box], models=[1])
    no_ops = {
        "no regions": lambda: sim.remove_particles([]),
        "region hits nothing": lambda: sim.remove_particles([objects.sphere((0.9, 0.9, 0.9), 0.01)]),
        "outside of everything": lambda: sim.remove_particles([objects.box((0.0, 0.0, 0.0), (1.0, 1.0, 1.0))], outside=True),
        "zero mask": lambda: sim.remove_rows(0, np.zeros(n, bool)),
    }
    for name, fn in no_ops.items():
        assert fn() == [0], name
        assert sim.save_checkpoint().tobytes() == before.tobytes(), name
    assert sim.counts[0] == n
    sim.step(5)
    assert sim.stats().error == 0
    sim.close()


def test_mgsp_is_not_supported(cuda_lib):
    pos = S.box(DX, (20, 20, 20), (24, 24, 24))
    ranks = [GmpmSimulator(dt=1e-4, fps=0, config=Config(domain_bits=6), max_blocks=4000, mgsp_world=2, mgsp_rank=r, auto_grow=False) for r in range(2)]
    ptrs = [s.mgsp_inbox() for s in ranks]
    for s in ranks:
        s.mgsp_set_peers(ptrs)
        s.init_model(S.FIXED_COROTATED, pos, (0, 0, 0))
    for s in ranks:
        with pytest.raises(CB200Error, match="CUDA error 801 "):
            s.remove_particles([objects.sphere((0.34, 0.34, 0.34), 0.02)])
        with pytest.raises(CB200Error, match="CUDA error 801 "):
            s.remove_rows(0, np.zeros(len(pos), bool))
        s.close()


def test_inflight_checkpoint_and_frame_deliver_the_state_before(cuda_lib, tmp_path):
    sim = S.build_engine(_odd_cube(S.J_FLUID))
    sim.step(4)
    want = sim.save_checkpoint()
    n = len(sim.retrieve(0))
    sim.checkpoint_begin()
    gone = sim.remove_particles([objects.box(np.array([20.0, 20.0, 20.0]) * DX, np.array([25.0, 40.0, 40.0]) * DX)])[0]
    assert gone > 0
    assert sim.checkpoint_end().tobytes() == want.tobytes()
    sim.write_frame(str(tmp_path), 1)
    sim.remove_particles([objects.box(np.array([27.0, 0.0, 0.0]) * DX, np.array([40.0, 40.0, 40.0]) * DX)])
    sim.wait_output()
    assert len(bgeo.read(os.path.join(str(tmp_path), "model_id[0]_frame[1].bgeo"))["position"]) == n - gone
    sim.step(3)
    assert sim.stats().error == 0
    sim.close()


def test_scene_sinks_per_frame_and_resume(cuda_lib, tmp_path):
    """A source above a sink box: the per-frame counts follow both schedules, and a resume at frame 3 reproduces frames 4-6."""
    doc = {"simulation": {"fps": 240, "frames": 6, "default_dt": 1e-4},
           "models": [{"constitutive": "jfluid", "file": "box", "offset": [0.3, 0.5, 0.3], "span": [0.1, 0.1, 0.1], "velocity": [0, -1, 0],
                       "rho": 1e3, "volume": DX ** 3 / 8, "bulk_modulus": 4e4, "gamma": 7.15, "viscosity": 0.01,
                       "emit": {"start": 2, "every": 1, "fill": "all"}}],
           "sinks": [{"shape": "box", "offset": [0.3, 0.5, 0.3], "span": [0.1, 0.05, 0.1], "start": 3, "every": 2}]}
    sched = sink_schedule(doc)
    assert list(sched) == [3, 5]
    path = os.path.join(str(tmp_path), "scene.json")
    with open(path, "w") as f:
        json.dump(doc, f)
    out = os.path.join(str(tmp_path), "out")
    os.mkdir(out)
    cfg = Config(domain_bits=6)
    sim = parse_scene(path, config=cfg)
    counts = {}
    ck = os.path.join(str(tmp_path), "f3.ckpt")

    def on_frame(s, f):
        counts[f] = s.counts[0]
        if f == 3:
            s.save_checkpoint(ck)
    n0 = sim.counts[0]
    sim.main_loop(output=out, on_frame=on_frame)
    assert sim.stats().error == 0
    sim.close()
    prev = n0
    for f in range(1, 7):
        n = len(bgeo.read(os.path.join(out, f"model_id[0]_frame[{f}].bgeo"))["position"])
        assert n == counts[f], f"frame {f}"
        if f in sched:
            assert n < prev + (n0 if f >= 2 else 0), f"frame {f}: the sink removed nothing"
        else:
            assert n == prev + (n0 if f >= 2 else 0), f"frame {f}"
        prev = n
    out2 = os.path.join(str(tmp_path), "out2")
    os.mkdir(out2)
    r = parse_scene(path, config=cfg, resume=ck)
    r.main_loop(output=out2)
    r.close()
    assert sorted(os.listdir(out2)) == [f"model_id[0]_frame[{f}].bgeo" for f in (4, 5, 6)]
    for f in (4, 5, 6):
        assert len(bgeo.read(os.path.join(out2, f"model_id[0]_frame[{f}].bgeo"))["position"]) == counts[f], f"resumed frame {f}"
