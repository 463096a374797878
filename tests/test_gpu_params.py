"""GPU tests of the step driver around a material parameter change between sub-steps (cb200_sim_update_*_parameters).

Every sub-step after an update is checked against ref64 with the parameters in effect, by ref64_checks' loops and bounds: across
a reserve and an auto_grow growth, with profiling (stream launches) switched on and off, after a restore, on MGSP ranks.  A
checkpoint carries the new parameters (and not one made between checkpoint_begin and _end), an emission after an update
rasterises the new mass, an emptied model takes an update, and a refused call changes nothing.
"""
import numpy as np
import pytest

import ref64
import ref64_cases as S
from claymore_b200 import checkpoint
from claymore_b200._capi import CB200Error, check
from claymore_b200.simulator import GmpmSimulator
from ref64_checks import engine_substep_check, mgsp_substep_check
from test_gpu_checkpoint import _restored
from test_gpu_emit import _grid_against
from test_gpu_emit import _mid_run_case as _emit_case
from test_ref64_mgsp_cpu import split_case

pytestmark = pytest.mark.gpu

DX = 1.0 / 64
GRAPH = pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])


def _floor_update(k=3, steps=(), rho=2.5e3, args=(2e4, 0.3)):
    """fixed-corotated on the floor: rho at sub-step k, E and nu at k + 3 (odd and even when k is odd), and ``steps`` checked.  In
    the first sub-steps the floor band's edge runs through the column, which takes even the FP32 oracle past KAPPA's F (as on
    walls_boundary1): these early sub-steps are held to the boundary bounds."""
    c = S._floor(S.FIXED_COROTATED, [])
    v = c["models"][0]["vol"]
    return dict(S._updated(c, {k: [(0, rho, v, (5e3, 0.4))], k + 3: [(0, rho, v, args)]}, list(steps)), boundary_bounds=True)


def _with_params(case, params):
    """``case`` with model i's (rho, vol, args) = params[i] (the parameters a restored simulator must carry)."""
    return dict(case, models=[dict(m, rho=p[0], vol=p[1], args=tuple(p[2])) for m, p in zip(case["models"], params)])


def _new_params(case):
    """A change of every parameter group of every model of ``case`` (rho x 1.5, vol x 0.75, each argument x 1.25)."""
    return [(m["rho"] * 1.5, m["vol"] * 0.75, tuple(a * 1.25 if i != 1 or m["material"] == S.J_FLUID else a * 0.8 for i, a in enumerate(m["args"])))
            for m in case["models"]]


def _mid_run_case():
    """test_gpu_emit's four materials; its sand starts on the cone tip (F = I), so every sand particle is near a branch point."""
    return dict(_emit_case(), max_near_branch=1.0)


def _update(sim, case, params):
    for i, (m, (rho, vol, args)) in enumerate(zip(case["models"], params)):
        getattr(sim, S.SETTER[m["material"]])(rho, vol, *args, model=i)


# ---- growth -----------------------------------------------------------------------------------------------------------------
def test_update_then_reserve(cuda_lib):
    """Graph mode: an update, then reserve (which re-creates every buffer and graph); every sub-step after both matches ref64."""
    case = _floor_update(steps=range(3, 10))
    grown = []

    def grow(sim, k):
        if k == 5:
            sim.reserve(sim.capacity()[0] * 2)
            grown.append(sim.capacity()[0])
    engine_substep_check(case, True, "update then reserve", before_step=grow)
    assert grown


def test_update_then_auto_grow(cuda_lib):
    """Graph mode: an update at sub-step 1 of a simulator 80 % full at the start (over auto_grow's 3/4): the capacity poll of the
    first sub-steps grows it after the update, at a sub-step the caller does not choose; every sub-step from 1 to 8 matches ref64."""
    case = _floor_update(k=1, steps=range(1, 9))
    probe = S.build_engine(case)
    ebc0 = probe.stats().exterior_block_count
    probe.close()
    sim = GmpmSimulator(dt=case["dt"], fps=0, config=S.config(case), max_blocks=int(ebc0 * 1.25), use_graph=True, auto_grow=True)
    for m in case["models"]:
        mid = sim.init_model(m["material"], m["pos"], m["v0"])
        getattr(sim, S.SETTER[m["material"]])(m["rho"], m["vol"], *m["args"], model=mid)
    sim.initial_setup()
    cap0, _ = sim.capacity()
    seen = {}

    def record(s, k):
        seen[k] = s.capacity()[0]
    engine_substep_check(case, True, "update then auto_grow", sim=sim, before_step=record)
    assert seen[1] == cap0 and seen[8] > cap0, (cap0, seen)


# ---- profiling ---------------------------------------------------------------------------------------------------------------
def test_update_while_profiling_then_graphs(cuda_lib):
    """Two graph sub-steps (the graphs exist), profiling on (stream launches), an update at sub-step 3, profiling off at sub-step 5
    (graph launches again): every sub-step from 3 matches ref64."""
    case = _floor_update(steps=range(3, 9))
    sim = S.build_engine(case, use_graph=True)
    sim.step(2)
    sim.profile(True)

    def toggle(s, k):
        if k == 5:
            s.profile(False)
    engine_substep_check(case, True, "update while profiling", sim=sim, before_step=toggle, start=2)


# ---- checkpoint ----------------------------------------------------------------------------------------------------------------
# checkpoint fields ref64.params sets; bm is a NACC parameter (the fixed-corotated and sand setters leave it alone, as the reference)
def _record_matches(record, material, params, label):
    want = ref64.params(material, params[0], params[1], *params[2])
    for f, v in want.items():
        if f == "material" or (f == "bm" and material != S.NACC):
            continue
        got = record[f]
        if isinstance(v, bool):
            assert int(got) == int(v), f"{label}: {f}"
        else:
            assert np.float32(got).tobytes() == np.float32(v).tobytes(), f"{label}: {f} {got!r} != {v!r}"


@GRAPH
def test_checkpoint_after_an_update(cuda_lib, use_graph):
    """Every model of every material updated after sub-step 4: the blob's parameter record is ref64.params of the new values, bit for
    bit; a restore of it then matches ref64 with the new parameters at sub-steps 4 and 5; an update between checkpoint_begin and
    checkpoint_end is not in that blob."""
    case = _mid_run_case()
    sim = S.build_engine(case, use_graph=use_graph)
    sim.step(4)
    new = _new_params(case)
    _update(sim, case, new)
    blob = sim.save_checkpoint()
    inf = checkpoint.info(blob)
    for i, m in enumerate(case["models"]):
        _record_matches(inf["models"][i]["params"], m["material"], new[i], f"model {i}")
    sim.checkpoint_begin()
    _update(sim, case, _new_params(_with_params(case, new)))
    during = sim.checkpoint_end()
    assert during.tobytes() == blob.tobytes()
    sim.close()
    r = _restored(blob, use_graph=use_graph)
    engine_substep_check(dict(_with_params(case, new), steps=[4, 5]), use_graph, "restored after an update", sim=r, start=4)


# ---- emission ----------------------------------------------------------------------------------------------------------------
@GRAPH
def test_emission_after_an_update_has_the_new_mass(cuda_lib, use_graph):
    case = _mid_run_case()
    sim = S.build_engine(case, use_graph=use_graph)
    sim.step(6)
    new = _new_params(case)
    _update(sim, case, new)
    a = checkpoint.read(sim.save_checkpoint())
    v = (0.0, -2.0, 0.5)
    pos = [S.box(DX, (14 + 8 * i, 46, 40), (18 + 8 * i, 50, 44)) for i in range(4)]
    for i, p in enumerate(pos):
        assert sim.add_particles(i, p, v) == len(p)
    masses = [S.ref_params(m)["mass"] for m in _with_params(case, new)["models"]]
    assert all(x != S.ref_params(m)["mass"] for x, m in zip(masses, case["models"]))
    _grid_against(sim, a["keys"], a["grid"], [dict(pos=p, v0=v, mass=x) for p, x in zip(pos, masses)], "grid after the emission")
    sim.close()


@GRAPH
def test_update_of_an_emptied_model(cuda_lib, use_graph):
    """A model emptied by removal takes an update; a later emission into it rasterises the new mass, and the sub-step after it
    matches ref64."""
    case = _mid_run_case()
    sim = S.build_engine(case, use_graph=use_graph)
    sim.step(3)
    sim.remove_rows(2, np.ones(len(sim.particle_state(2)), bool))
    assert len(sim.particle_state(2)) == 0
    m = case["models"][2]
    new = (2e3, m["vol"] * 0.5, (2e4, 0.3))
    sim.update_fr_parameters(*new[:2], *new[2], model=2)
    sim.step(2)
    g = sim.grid()
    keys, grid = sim.active_keys()[: len(g)].copy(), g.copy()
    p = S.box(DX, (38, 20, 22), (42, 24, 26))
    v = (0.0, -1.0, 0.0)
    assert sim.add_particles(2, p, v) == len(p)
    mass = ref64.params(m["material"], new[0], new[1], *new[2])["mass"]
    _grid_against(sim, keys, grid, [dict(pos=p, v0=v, mass=mass)], "emission into the emptied model")
    models = [dict(x, pos=sim.particle_state(i)[:, :3]) for i, x in enumerate(case["models"])]
    models[2].update(rho=new[0], vol=new[1], args=new[2])
    engine_substep_check(dict(case, models=models, steps=[5, 6]), use_graph, "after the emission into the emptied model", sim=sim, start=5)


# ---- MGSP ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(600)
@GRAPH
@pytest.mark.parametrize("world,kind", [(2, "x"), (4, "2x2")], ids=["2x", "2x2"])
def test_mgsp_ranks_take_the_same_update(cuda_lib, world, kind, use_graph):
    """Every rank makes the same setter calls between sub-steps (rank_update): rho at 1, E and nu at 4."""
    case = _floor_update(k=1, steps=range(1, 7))
    parts = split_case(case, world, kind)
    mgsp_substep_check(case, parts, use_graph, f"update on {world} ranks {kind} {'graph' if use_graph else 'stream'}")


# ---- rejections and what a valid update keeps -------------------------------------------------------------------------------
def test_rejections_leave_the_simulator_unchanged(cuda_lib):
    case = S._cube(S.FIXED_COROTATED, steps=[])
    empty = GmpmSimulator(dt=1e-4, fps=0, config=S.config(case), max_blocks=1000)
    for setter, args in (("update_fr_parameters", (1e3, 1e-6, 5e3, 0.4)), ("update_j_fluid_parameters", (1e3, 1e-6, 4e4, 7.15, 0.01))):
        with pytest.raises(CB200Error, match="CUDA error 1 "):   # no model yet
            getattr(empty, setter)(*args, model=0)
    empty.close()
    sim = S.build_engine(case)
    sim.step(4)
    before = sim.save_checkpoint()
    bad_calls = {
        "fluid setter on a fixed-corotated model": lambda: sim.update_j_fluid_parameters(2e3, 1e-6, 4e4, 7.15, 0.01, model=0),
        "sand setter on a fixed-corotated model": lambda: sim.update_sand_parameters(2e3, 1e-6, 5e3, 0.4, model=0),
        "NACC setter on a fixed-corotated model": lambda: sim.update_nacc_parameters(2e3, 1e-6, 5e3, 0.4, 0.5, 0.8, model=0),
        "model 1 of 1": lambda: sim.update_fr_parameters(2e3, 1e-6, 5e3, 0.4, model=1),
        "model 8": lambda: sim.update_fr_parameters(2e3, 1e-6, 5e3, 0.4, model=8),
        "model -2": lambda: check(sim.L.cb200_sim_update_fr_parameters(sim.h, -2, 2e3, 1e-6, 5e3, 0.4), "update_fr_parameters"),
    }
    for name, fn in bad_calls.items():
        with pytest.raises(CB200Error, match="CUDA error 1 "):
            fn()
        assert sim.save_checkpoint().tobytes() == before.tobytes(), name
    sim.step(3)
    assert sim.stats().error == 0
    sim.close()


def test_a_valid_update_keeps_the_force_report_and_the_clock(cuda_lib):
    """The force report (sums and the span they cover) and the clock run on through an update that keeps the values: a run with
    the update equals a run without it."""
    case = S.OBJECT_CASES["obj_floor_fc_sticky"]
    m = case["models"][0]
    out = []
    for update in (False, True):
        sim = S.build_engine(case)
        sim.report_forces(True)
        sim.step(14)
        t = sim.sim_time()
        if update:
            sim.update_fr_parameters(m["rho"], m["vol"], *m["args"], model=0)
        assert sim.sim_time() == t
        sim.step(14)
        out.append((sim.sim_time(), *sim.collision_forces()))
        sim.close()
    (t0, e0, j0), (t1, e1, j1) = out
    assert t1 == t0 and e1 == e0 > 0, (t0, t1, e0, e1)
    assert np.abs(j0).max() > 0 and np.abs(j1 - j0).max() <= 1e-5 * np.abs(j0).max(), (j0, j1)
