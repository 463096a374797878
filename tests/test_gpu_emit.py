"""GPU tests of adding particles to a set-up simulator (cb200_sim_add_particles / _add_particles_sdf, GmpmSimulator.add_particles,
the scene's "emit").

Right after initial_setup an emission equals a set-up over the union (keys, rows, dt bitwise; grid within the rasterisation bound of
ref64).  Mid-run, the rows and keys are those of the state before plus the new particles, grid[0] gains exactly their
rasterisation, and the next sub-step matches ref64.  Every rejection leaves a checkpoint byte-identical to the one before it.
"""
import json
import os

import numpy as np
import pytest

import ref64
import ref64_cases as S
import scenes
from claymore_b200 import bgeo, checkpoint
from claymore_b200._capi import CB200Error, Config
from claymore_b200.scene import emit_schedule, parse_scene
from claymore_b200.simulator import GmpmSimulator
from ref64_checks import BRANCH_MARGIN, F_ALLOW, KAPPA, RASTER_KAPPA, STRESS_ALLOW, check_counts, check_dt, check_report, ref_models
from test_gpu_checkpoint import _assert_round_trip, _restored, _sorted_rows
from test_gpu_parity import _compare_state

pytestmark = pytest.mark.gpu

DX = 1.0 / 64
MATERIALS = [S.FIXED_COROTATED, S.J_FLUID, S.SAND, S.NACC]
EPS = 2.0 ** -24


def _new_rows(material, pos):
    """What array_to_buffer starts a particle from: position, F = I (J = 1), logJp = LOG_JP_0."""
    pos = np.asarray(pos, np.float32)
    if material == S.J_FLUID:
        return np.concatenate([pos, np.ones((len(pos), 1), np.float32)], 1)
    rows = np.concatenate([pos, np.tile(np.eye(3, dtype=np.float32).reshape(1, 9), (len(pos), 1))], 1)
    if material == S.FIXED_COROTATED:
        return rows
    return np.concatenate([rows, np.full((len(pos), 1), 0.0 if material == S.SAND else -0.01, np.float32)], 1)


def _key_classes(sim):
    st = sim.stats()
    k = sim.active_keys()
    b = (0, st.particle_block_count, st.neighbor_block_count, st.exterior_block_count)
    return [np.sort(scenes.key_hash(k[lo:hi])) for lo, hi in zip(b[:-1], b[1:])]


def _assert_same_classes(a, b, label):
    for i, (x, y) in enumerate(zip(_key_classes(a), _key_classes(b))):
        assert np.array_equal(x, y), f"{label}: key class {i}"


def _grid_against(sim, base_keys, base_grid, new_models, label):
    """sim's grid[0] per cell == base (by key, 0 for new blocks) + ref64.rasterize(new_models), within RASTER_KAPPA of the new
    contribution plus the one float32 rounding of the sum."""
    st = sim.stats()
    keys, grid = sim.active_keys()[: st.neighbor_block_count], sim.grid()
    rk, rg, rmag = ref64.rasterize(sim.cfg, new_models)
    h = scenes.key_hash(keys)
    pos = {int(x): i for i, x in enumerate(h)}
    expect = np.zeros(grid.shape, np.float64)
    mag = np.zeros(grid.shape, np.float64)
    if base_keys is not None:
        for k, g in zip(scenes.key_hash(base_keys), base_grid):
            assert int(k) in pos, f"{label}: a block of the state before is missing"
            expect[pos[int(k)]] += g
    for k, g, m in zip(scenes.key_hash(rk), rg, rmag):
        if int(k) not in pos:   # beyond the top face: dropped
            continue
        expect[pos[int(k)]] += g
        mag[pos[int(k)]] += m
    err = np.abs(grid.astype(np.float64) - expect)
    tol = RASTER_KAPPA["mass"] * EPS * mag + EPS * np.abs(expect) + 1e-30
    assert (err <= tol).all(), f"{label}: grid off by {(err / tol).max():.3g} x its bound"


def _mass(material):
    return S.ref_params(S.model(material, np.zeros((1, 3)), (0, 0, 0), DX))["mass"]


@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
@pytest.mark.parametrize("material", MATERIALS)
def test_emission_after_setup_equals_setup_over_the_union(cuda_lib, material, use_graph):
    v = (0.3, -1.0, 0.2)
    p1, p2 = S.box(DX, (20, 20, 20), (32, 32, 32)), S.box(DX, (22, 34, 22), (30, 40, 30))
    one = S.build_engine(S._case(6, [S.model(material, p1, v, DX)], []), use_graph=use_graph)
    assert one.add_particles(0, p2, v) == len(p2)
    both = S.build_engine(S._case(6, [S.model(material, np.concatenate([p1, p2]), v, DX)], []), use_graph=use_graph)
    assert one.counts[0] == len(p1) + len(p2)
    _assert_same_classes(one, both, "emission vs set-up over the union")
    assert _sorted_rows(one.particle_state(0)).tobytes() == _sorted_rows(both.particle_state(0)).tobytes()
    sa, sb = one.stats(), both.stats()
    assert (sa.dt, sa.next_dt, sa.steps, sa.error) == (sb.dt, sb.next_dt, 0, 0)
    _grid_against(one, None, None, [dict(pos=np.concatenate([p1, p2]), v0=v, mass=_mass(material))], "union rasterisation")
    one.step(20)
    both.step(20)
    _compare_state(both, one, 1, "20 sub-steps after the emission", pos_tol=5e-6, f_tol=2e-4)
    one.close()
    both.close()


def _mid_run_case():
    dx = DX
    ms = [S.model(S.J_FLUID, S.box(dx, (14, 20, 20), (22, 28, 28)), (0.5, -0.5, 0.0), dx),
          S.model(S.SAND, S.box(dx, (26, 22, 20), (34, 30, 28)), (0.0, -0.8, 0.2), dx),
          S.model(S.FIXED_COROTATED, S.box(dx, (38, 20, 22), (46, 28, 30)), (-0.5, -0.3, 0.0), dx),
          S.model(S.NACC, S.box(dx, (26, 36, 30), (32, 42, 36)), (0.0, -1.0, 0.0), dx)]
    return S._case(6, ms, [])


@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
def test_mid_run_emission_into_every_model(cuda_lib, use_graph):
    case = _mid_run_case()
    sim = S.build_engine(case, use_graph=use_graph)
    sim.step(10)
    a = checkpoint.read(sim.save_checkpoint())
    sa = sim.stats()
    v = (0.0, -2.0, 0.5)
    new = [S.box(DX, (14 + 8 * i, 46, 40), (18 + 8 * i, 50, 44)) for i in range(4)]
    for i, p in enumerate(new):
        assert sim.add_particles(i, p, v) == len(p)
    b = checkpoint.read(sim.save_checkpoint())
    for i, m in enumerate(case["models"]):
        want = _sorted_rows(np.concatenate([a["states"][i], _new_rows(m["material"], new[i])]))
        assert _sorted_rows(b["states"][i]).tobytes() == want.tobytes(), f"model {i} rows"
    fresh = S.build_engine(S._case(6, [dict(m, pos=b["states"][i][:, :3].copy()) for i, m in enumerate(case["models"])], []))
    _assert_same_classes(sim, fresh, "mid-run emission vs a set-up on B's positions")
    fresh.close()
    _grid_against(sim, a["keys"], a["grid"], [dict(pos=p, v0=v, mass=S.ref_params(m)["mass"]) for p, m in zip(new, case["models"])], "grid B - A")
    for f in ("steps", "sim_time", "step_time", "frame_time", "frames"):
        assert a[f] == b[f], f
    rule = np.float32(np.float32(DX) * np.float32(0.5) / np.sqrt(np.float32(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]), dtype=np.float32))
    assert b["dt"] == min(np.float32(sa.dt), rule) and b["next_dt"] == b["dt"]
    n_m = sum(len(p) * S.ref_params(m)["mass"] for p, m in zip(new, case["models"]))
    ga, gb = a["grid"].astype(np.float64), b["grid"].astype(np.float64)
    assert abs((gb[:, 0].sum() - ga[:, 0].sum()) - n_m) <= 1e-5 * gb[:, 0].sum()
    for d in range(3):
        assert abs((gb[:, 1 + d].sum() - ga[:, 1 + d].sum()) - n_m * v[d]) <= 1e-5 * abs(gb[:, 1 + d]).sum() + 1e-12
    # one sub-step from B against ref64: the rebuilt bins, buckets and tags are a valid start
    st = sim.stats()
    g = sim.grid()
    keys, before = sim.active_keys()[: len(g)], [sim.particle_state(i) for i in range(4)]
    r = ref64.substep(sim.cfg, ref_models(case, before), keys, g, st.dt, case["dt"])
    sim.step(1)
    assert sim.stats().error == 0
    g = sim.grid()
    states = [sim.particle_state(i) for i in range(4)]
    check_counts(r, before, states, case["max_ppc"], "sub-step after the emission")
    rep = ref64.compare(r, sim.active_keys()[: len(g)], g, states, KAPPA, STRESS_ALLOW, [F_ALLOW[m["material"]] for m in case["models"]], margin=BRANCH_MARGIN,
                        max_ppc=case["max_ppc"])
    check_report(rep, "sub-step after the emission")
    check_dt(sim.stats().dt, r["new_dt"], "sub-step after the emission")
    sim.close()


def test_dt_rule(cuda_lib):
    sim = S.build_engine(S._cube(S.FIXED_COROTATED, steps=[], dt=1e-3))   # dt_default above the CFL bound of the emission
    sim.step(3)
    before = sim.stats()
    t0 = sim.sim_time()
    v = np.float32([3.0, -10.0, 2.0])   # ten times the cube's v0
    sim.add_particles(0, S.box(DX, (22, 36, 22), (26, 40, 26)), v)
    rule = np.float32(DX) * np.float32(0.5) / np.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])
    st = sim.stats()
    assert rule < np.float32(before.dt)
    assert st.dt == rule and st.next_dt == st.dt and st.steps == before.steps
    assert sim.sim_time() == t0
    sim.step(1)
    assert sim.sim_time() == t0 + float(np.float32(st.dt))
    sim.close()


def _cell(x):
    """cell_index: the float32 product x * 2^bits rounded half away from zero"""
    p = np.asarray(x, np.float32) * np.float32(64)
    return (np.sign(p) * np.floor(np.abs(p) + np.float32(0.5))).astype(np.int64)


def test_empty_cell_filter(cuda_lib):
    sim = S.build_engine(S._cube(S.J_FLUID, v0=(0.0, -1.0, 0.0), steps=[]))
    cand = S.box(DX, (18, 18, 18), (34, 34, 34))
    assert sim.add_particles(0, cand, fill="empty") > 0     # the shell around the cube
    assert sim.add_particles(0, cand, fill="empty") == 0   # the same region again at one boundary
    sim.step(15)
    assert sim.stats().error == 0
    occupied = {tuple(c) for c in _cell(sim.retrieve(0))}
    want = sum(tuple(c) not in occupied for c in _cell(cand))
    blob = sim.save_checkpoint()
    assert sim.add_particles(0, cand, fill="empty") == want
    assert sim.save_checkpoint().tobytes() != blob.tobytes() or want == 0
    sim.step(5)
    assert sim.stats().error == 0
    sim.close()


def _cell_centres(lo, hi):
    """one candidate at the centre of every cell of [lo, hi)^3 (cells), so every bucket cell of a block, (3, 3, 3) included, has one"""
    ax = [np.arange(l, h, dtype=np.float64) * DX for l, h in zip(lo, hi)]
    return np.stack(np.meshgrid(*ax, indexing="ij"), -1).reshape(-1, 3).astype(np.float32)


@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
def test_empty_cell_filter_with_models_parting_across_blocks(cuda_lib, use_graph):
    """Two models share the blocks at their interface, then move apart: blocks empty out, new ones appear and the partition is
    renumbered, so a block number that held one model's particles comes to hold only the other's.  The filter's count must still be
    the numpy count of candidates in cells no particle holds, and a cell that is full through one model must reject an overflow."""
    dx = DX
    fluid = S.model(S.J_FLUID, S.box(dx, (17, 22, 22), (29, 30, 30)), (-20.0, 0.0, 0.0), dx)   # bucket cells 15..26: shares blocks with
    sand = S.model(S.SAND, S.box(dx, (29, 22, 22), (41, 30, 30)), (20.0, 0.0, 0.0), dx)        # the sand's 27.. at the interface
    case = S._case(6, [fluid, sand], [])
    sim = S.build_engine(case, use_graph=use_graph)
    cand = _cell_centres((8, 18, 18), (52, 34, 34))
    sim.step(36)   # about 4.6 cells apart: blocks emptied, new blocks, renumbered partitions
    assert sim.stats().error == 0
    occupied = {tuple(c) for m in range(2) for c in _cell(sim.retrieve(m))}
    want = sum(tuple(c) not in occupied for c in _cell(cand))
    assert 0 < want < len(cand)
    assert sim.add_particles(1, cand, (0.0, 0.0, 0.0), fill="empty") == want
    assert sim.add_particles(1, cand, (0.0, 0.0, 0.0), fill="empty") == 0
    # a cell filled up to max_ppc through one model: one particle more is an overflow, rejected before anything changes
    p = sim.retrieve(0)[:1]
    cell = tuple(_cell(p)[0])
    have = sum(sum(tuple(c) == cell for c in _cell(sim.retrieve(m))) for m in range(2))
    blob = sim.save_checkpoint()
    with pytest.raises(CB200Error, match="CUDA error 1 "):
        sim.add_particles(0, np.repeat(p, case["max_ppc"] - have + 1, 0))
    assert sim.save_checkpoint().tobytes() == blob.tobytes()
    assert sim.add_particles(0, np.repeat(p, case["max_ppc"] - have, 0)) == case["max_ppc"] - have
    assert sim.stats().error == 0
    sim.close()


def test_empty_cell_filter_random_sdf_is_deterministic(cuda_lib):
    ls = _sphere_level_set()
    rows = []
    for _ in range(2):
        sim = S.build_engine(S._cube(S.SAND, steps=[]))
        sim.step(5)
        n = sim.add_particles_sdf(0, ls, (0.25, 0.25, 0.25), (0.5, 0.5, 0.5), (0.0, -1.0, 0.0), ppc=8, mode="random", seed=7, fill="empty")
        assert n > 0
        rows.append(_sorted_rows(sim.particle_state(0)))
        sim.close()
    assert rows[0].tobytes() == rows[1].tobytes()


def _sphere_level_set(n=21):
    from claymore_b200 import sdf as sdfmod
    q = np.linspace(-1.0, 1.0, n)
    x, y, z = np.meshgrid(q, q, q, indexing="ij")
    phi = (np.sqrt(x * x + y * y + z * z) - 0.8).astype(np.float32)
    text = f"{n} {n} {n}\n-1 -1 -1\n{2.0 / (n - 1)!r}\n" + "\n".join(repr(float(v)) for v in phi.transpose(2, 1, 0).ravel()) + "\n"
    return sdfmod.parse(text.encode())


def test_capacity(cuda_lib):
    case = S._cube(S.FIXED_COROTATED, steps=[])
    far = S.box(DX, (44, 44, 44), (52, 52, 52))
    sim = GmpmSimulator(dt=1e-4, fps=0, config=S.config(case), max_blocks=300, auto_grow=False)
    sim.init_model(S.FIXED_COROTATED, case["models"][0]["pos"], case["models"][0]["v0"])
    sim.initial_setup()
    sim.step(3)
    before = sim.save_checkpoint()
    with pytest.raises(CB200Error, match="CUDA error 2 "):
        sim.add_particles(0, far, (0, 0, 0))
    assert sim.save_checkpoint().tobytes() == before.tobytes()
    sim.step(5)
    assert sim.stats().error == 0
    sim.close()
    sim = GmpmSimulator(dt=1e-4, fps=0, config=S.config(case), max_blocks=300, auto_grow=True)
    sim.init_model(S.FIXED_COROTATED, case["models"][0]["pos"], case["models"][0]["v0"])
    sim.initial_setup()
    ev = sim.capacity()[1]
    assert sim.add_particles(0, far, (0, 0, 0)) == len(far)
    assert sim.capacity()[1] > ev
    sim.step(5)
    assert sim.stats().error == 0
    sim.close()
    # doubling a model grows its bins (too few set kErrBinCapacity); the sub-steps after run clean
    sim = S.build_engine(case)
    pos = case["models"][0]["pos"]
    assert sim.add_particles(0, pos + np.float32([0.0, 14 * DX, 0.0]), case["models"][0]["v0"]) == len(pos)
    assert sim.counts[0] == 2 * len(pos) == len(sim.retrieve(0))
    sim.step(20)
    assert sim.stats().error == 0
    sim.close()


def test_rejections_leave_the_simulator_unchanged(cuda_lib):
    case = S._cube(S.FIXED_COROTATED, steps=[])
    pos = case["models"][0]["pos"]
    fresh = GmpmSimulator(dt=1e-4, fps=0, config=S.config(case), max_blocks=4000)
    fresh.init_model(S.FIXED_COROTATED, pos, (0, 0, 0))
    with pytest.raises(CB200Error, match="CUDA error 1 "):       # not set up
        fresh.add_particles(0, pos[:10])
    fresh.close()
    sim = S.build_engine(case)
    sim.step(4)
    before = sim.save_checkpoint()
    ok = S.box(DX, (22, 36, 22), (24, 38, 24))
    dense = np.repeat(ok[:1], 129, 0)
    bad_calls = {
        "bad model": lambda: sim.add_particles(3, ok),
        "negative model": lambda: sim.add_particles(-1, ok),
        "nan": lambda: sim.add_particles(0, np.concatenate([ok, [[np.nan, 0.5, 0.5]]])),
        "inf": lambda: sim.add_particles(0, np.concatenate([ok, [[0.5, np.inf, 0.5]]])),
        "outside low": lambda: sim.add_particles(0, np.concatenate([ok, [[0.5, 1.4 * DX, 0.5]]])),
        "outside high": lambda: sim.add_particles(0, np.concatenate([ok, [[0.5, 1.0 + 2.0 * DX, 0.5]]])),
        "cell overflow": lambda: sim.add_particles(0, dense),
        "cell overflow with existing": lambda: sim.add_particles(0, np.repeat(pos[:1], 128, 0)),
        "flags": lambda: sim.L.cb200_sim_add_particles(sim.h, 0, ok.ctypes.data_as(type(sim.h)), len(ok), None, 6, None),
        "nan v0": lambda: sim.add_particles(0, ok, (0.0, np.nan, 0.0)),
        "inf v0": lambda: sim.add_particles(0, ok, (np.inf, 0.0, 0.0)),
    }
    for name, fn in bad_calls.items():
        if name == "flags":
            assert fn() == 1, name
        else:
            with pytest.raises(CB200Error, match="CUDA error 1 "):
                fn()
        assert sim.save_checkpoint().tobytes() == before.tobytes(), name
    with pytest.raises(ValueError):
        sim.add_particles(0, ok, fill="most")
    for v in ((1.0, 2.0), (1.0, 2.0, 3.0, 4.0), [[0.0, 0.0, 0.0]]):   # the library reads three floats
        with pytest.raises(ValueError, match="v0"):
            sim.add_particles(0, ok, v)
    assert sim.add_particles(0, ok[:0]) == 0
    assert sim.save_checkpoint().tobytes() == before.tobytes()
    sim.step(5)
    assert sim.stats().error == 0
    sim.close()


def test_mgsp_is_not_supported(cuda_lib):
    """Two in-process ranks wired to each other: both refuse with cudaErrorNotSupported, as cb200_sim_reserve does."""
    pos = S.box(DX, (20, 20, 20), (24, 24, 24))
    ranks = [GmpmSimulator(dt=1e-4, fps=0, config=Config(domain_bits=6), max_blocks=4000, mgsp_world=2, mgsp_rank=r, auto_grow=False) for r in range(2)]
    ptrs = [s.mgsp_inbox() for s in ranks]
    for s in ranks:
        s.mgsp_set_peers(ptrs)
        s.init_model(S.FIXED_COROTATED, pos, (0, 0, 0))
    for s in ranks:
        with pytest.raises(CB200Error, match="CUDA error 801 "):
            s.add_particles(0, pos[:8])
        s.close()


def test_inflight_checkpoint_and_frame_deliver_the_state_before(cuda_lib, tmp_path):
    sim = S.build_engine(S._cube(S.J_FLUID, steps=[]))
    sim.step(4)
    want = sim.save_checkpoint()
    sim.checkpoint_begin()
    add = S.box(DX, (22, 36, 22), (26, 40, 26))
    sim.add_particles(0, add, (0.0, -1.0, 0.0))
    assert sim.checkpoint_end().tobytes() == want.tobytes()
    n_before = len(sim.retrieve(0)) - len(add)
    sim.write_frame(str(tmp_path), 1)
    sim.add_particles(0, S.box(DX, (22, 42, 22), (26, 46, 26)), (0.0, -1.0, 0.0))
    sim.wait_output()
    assert len(bgeo.read(os.path.join(str(tmp_path), "model_id[0]_frame[1].bgeo"))["position"]) == n_before + len(add)
    # a checkpoint after an emission restores exactly
    blob = sim.save_checkpoint()
    r = _restored(blob)
    _assert_round_trip(sim, r, 1)
    r.step(3)
    sim.step(3)
    _compare_state(sim, r, 1, "3 sub-steps after a restore of an emission", pos_tol=5e-6, f_tol=2e-4)
    r.close()
    sim.close()


def test_scene_emits_per_frame_and_resumes(cuda_lib, tmp_path):
    doc = {"simulation": {"fps": 240, "frames": 6, "default_dt": 1e-4},
           "models": [{"constitutive": "jfluid", "file": "box", "offset": [0.3, 0.5, 0.3], "span": [0.1, 0.1, 0.1], "velocity": [0, -1, 0],
                       "rho": 1e3, "volume": DX ** 3 / 8, "bulk_modulus": 4e4, "gamma": 7.15, "viscosity": 0.01,
                       "emit": {"start": 2, "every": 2, "fill": "all"}}]}
    sched = emit_schedule(doc)[0]
    assert [f for f, _ in sched] == [2, 4, 6]
    path = os.path.join(str(tmp_path), "scene.json")
    with open(path, "w") as f:
        json.dump(doc, f)
    out = os.path.join(str(tmp_path), "out")
    os.mkdir(out)
    cfg = Config(domain_bits=6)
    sim = parse_scene(path, config=cfg)
    n0 = sim.counts[0]
    ck = os.path.join(str(tmp_path), "f3.ckpt")
    sim.main_loop(output=out, on_frame=lambda s, f: s.save_checkpoint(ck) if f == 3 else None)
    assert sim.stats().error == 0
    sim.close()
    total, counts = n0, {}
    for f in range(1, 7):
        if f in dict(sched):
            total += n0
        counts[f] = total
        assert len(bgeo.read(os.path.join(out, f"model_id[0]_frame[{f}].bgeo"))["position"]) == total, f"frame {f}"
    out2 = os.path.join(str(tmp_path), "out2")
    os.mkdir(out2)
    r = parse_scene(path, config=cfg, resume=ck)
    r.main_loop(output=out2)
    assert r.counts[0] == counts[6]
    r.close()
    assert sorted(os.listdir(out2)) == [f"model_id[0]_frame[{f}].bgeo" for f in (4, 5, 6)]
    for f in (4, 5, 6):
        assert len(bgeo.read(os.path.join(out2, f"model_id[0]_frame[{f}].bgeo"))["position"]) == counts[f], f"resumed frame {f}"
