"""The engine's signed-distance collider against the float64 reference (ref64.collider_resolve), with the kappa values
test_ref64_collider_cpu.py fixed on the FP32 collider oracle (no re-tuning here).

Kernel level: cb200_update_grid_velocity_query_max_collider on the synthetic grids and parameter matrix of the CPU test, per
node.  Step driver: every case of COLLIDER_CASES in graph and stream mode, one sub-step at a time, the collider placed at the
simulated time the engine reports before the sub-step.  MGSP: the ranks' dt comes from the max their next-max predictor
(carry_grid_boundary_kernel, grid_max_boundary_kernel at set-up) computed for the next grid update; it must be bit-identical on
every rank and within DT_ULPS of ref64's grid update at that time.
"""
import ctypes as C

import numpy as np
import pytest

import ref64
import ref64_cases as S
import ref64_mgsp as M
from test_gpu_mgsp_ref64 import on_threads
from test_ref64_collider_cpu import (COLLIDER_KAPPA, FIELDS, KERNEL_MATRIX, block_field, check_dt_range, collider_report, kernel_matrix,
                                     new_counts, substep_compare)
from test_ref64_cpu import BRANCH_MARGIN, F_ALLOW, RASTER_KAPPA, STRESS_ALLOW, check_report, ref_models
from test_ref64_mgsp_cpu import rank_models, split_case

pytestmark = pytest.mark.gpu

ERR_LOST, ERR_CELL_OVERFLOW = 4, 8


# ---- kernel level ---------------------------------------------------------------------------------------------------------
def engine_kernel(cuda_lib):
    import torch
    from claymore_b200._capi import Collider, Config, Partition
    cache = {}

    def run(cfg, keys, grid, dt, spec, t):
        key = (cfg.domain_bits, repr(spec_field[0]))
        if key not in cache:
            cache.clear()
            sdf, grad = S.make_field(cfg.domain_bits, spec_field[0])
            cache[key] = torch.from_numpy(block_field(cfg.domain_bits, sdf, grad)).cuda()
        col = S.collider_struct(Collider(), spec)
        col.sdf = cache[key].data_ptr()
        g = torch.from_numpy(np.ascontiguousarray(grid)).cuda()
        k = torch.from_numpy(np.ascontiguousarray(keys.reshape(-1))).cuda()
        mv = torch.zeros(1, dtype=torch.float32, device="cuda")
        part = Partition()
        part.active_keys = k.data_ptr()
        ecfg = Config(domain_bits=cfg.domain_bits, boundary=cfg.boundary, gravity=cfg.gravity)
        assert cuda_lib.cb200_update_grid_velocity_query_max_collider(C.byref(ecfg), len(keys), C.c_void_p(g.data_ptr()), part, dt, C.byref(col),
                                                                      float(np.float32(t)), C.c_void_p(mv.data_ptr()), None) == 0
        torch.cuda.synchronize()
        return g.cpu().numpy(), float(mv.item())
    spec_field = [None]
    return run, spec_field


@pytest.mark.parametrize("field,boundary,motion", KERNEL_MATRIX, ids=[f"{f}-b{b}-{m}" for f, b, m in KERNEL_MATRIX])
def test_engine_collider_kernel_matches_ref64(oracle, cuda_lib, field, boundary, motion):
    run, spec_field = engine_kernel(cuda_lib)
    spec_field[0] = FIELDS[field]
    worst, near, total, _ = kernel_matrix(run, oracle, field, boundary, motion, f"cb200 {field} boundary {boundary} {motion}")
    print(f"cb200 {field} boundary {boundary} {motion}: worst {worst:.3f} x COLLIDER_VEL_KAPPA, {near} of {total} nodes near")


# ---- step driver ----------------------------------------------------------------------------------------------------------
def _engine_state(sim, nm):
    g = sim.grid()
    return sim.active_keys()[: len(g)], g, [sim.particle_state(i) for i in range(nm)]


def engine_collider_check(case, use_graph, label):
    sim = S.build_engine(case, use_graph=use_graph)
    ccol, objs = S.ref_collider(case), S.ref_objects(case)
    nm = len(case["models"])
    done, expect = 0, 0
    counts = new_counts()
    for k in case["steps"]:
        sim.step(k - done)
        st = sim.stats()
        assert st.error == expect, f"{label}: error bits {st.error} at sub-step {k}, expected {expect}"
        keys, grid, before = _engine_state(sim, nm)
        t = sim.sim_time()
        r = ref64.substep(sim.cfg, ref_models(case, before), keys, grid, st.dt, case["dt"], S.engine_time_left(sim, case), ccol,
                          np.float32(t) if ccol is not None or objs else 0.0, objects=objs)
        sim.step(1)
        done = k + 1
        assert sim.sim_time() == t + float(np.float32(st.dt)), f"{label}: sim_time {sim.sim_time()!r} after a sub-step of {st.dt!r} from {t!r}"
        st = sim.stats()
        if any(m["dropped"].any() or m["lost"].any() for m in r["models"]):
            expect |= ERR_LOST
        if any(ref64.cell_overflow(m, case["max_ppc"])[1] for m in r["models"]):
            expect |= ERR_CELL_OVERFLOW
        assert st.error == expect, f"{label}: error bits {st.error} after sub-step {k}, expected {expect}"
        keys, grid, states = _engine_state(sim, nm)
        substep_compare(case, r, keys, grid, before, states, st.dt, f"{label} sub-step {k}", counts)
    sim.close()
    collider_report(case, label, counts)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
@pytest.mark.parametrize("name", list(S.COLLIDER_CASES))
def test_engine_collider_substep_matches_ref64(cuda_lib, name, use_graph):
    engine_collider_check(S.COLLIDER_CASES[name], use_graph, f"{name} {'graph' if use_graph else 'stream'}")


# ---- MGSP -------------------------------------------------------------------------------------------------------------------
def build_ranks_with_collider(case, parts, use_graph, max_blocks=6000):
    """The ranks of test_gpu_mgsp_ref64.build_ranks with the case's collider and objects set before initial_setup, so that the
    set-up's next-max predictor (grid_max_boundary_kernel) applies them."""
    from claymore_b200.simulator import GmpmSimulator
    sims = []
    for r, ps in enumerate(parts):
        sim = GmpmSimulator(dt=case["dt"], fps=case.get("fps", 0), config=S.config(case), max_blocks=max_blocks, use_graph=use_graph,
                            mgsp_rank=r, mgsp_world=len(parts))
        for q in ps:
            mid = sim.init_model(q["material"], q["pos"], q["v0"])
            getattr(sim, S.SETTER[q["material"]])(q["rho"], q["vol"], *q["args"], model=mid)
        if case.get("collider"):
            sdf, grad = S.collider_field(case)
            p = S.collider_spec(case["collider"])
            sim.set_collider(sdf, grad, type=p["type"], friction=p["friction"], trans=p["trans"], trans_vel=p["trans_vel"], omega=p["omega"],
                             rot=np.asarray(p["rot_mat"]).reshape(3, 3), scale=p["scale"], dsdt=p["dsdt"])
        if case.get("objects"):
            sim.set_collision_objects(S.object_structs(case))
        sims.append(sim)
    ptrs = [s.mgsp_inbox() for s in sims]
    for s in sims:
        s.mgsp_set_peers(ptrs)
    on_threads(sims, lambda s: s.initial_setup())
    return sims


def _grid(sim):
    g = sim.grid()
    return sim.active_keys()[: len(g)].astype(np.int64), g


def mgsp_collider_check(case, parts, use_graph, label):
    """Set-up grid and case['steps'] sub-steps of the ranks against ref64_mgsp with the collider at the engine's sim_time;
    sub-step 0's dt is the set-up predictor's (grid_max_boundary_kernel at t = 0), every later one the carry kernel's."""
    sims = build_ranks_with_collider(case, parts, use_graph)
    cfg = sims[0].cfg
    ccol, objs = S.ref_collider(case), S.ref_objects(case)
    nm = len(case["models"])
    for s in sims:
        assert s.stats().error == 0
    ref = M.rasterize(cfg, [[dict(pos=p["pos"], v0=p["v0"], mass=S.ref_params(p)["mass"]) for p in ps] for ps in parts])
    check_report(M.compare(cfg, ref, [dict(zip(("keys", "grid"), _grid(s))) for s in sims], RASTER_KAPPA, 0.0, []), f"{label} set-up")
    done, near, tainted = 0, 0, 0
    f_allow = [F_ALLOW[m["material"]] for m in case["models"]]
    for k in case["steps"]:
        if k > done:
            on_threads(sims, lambda s: (s.step(k - done), s.sync()))
        ranks = []
        for s, ps in zip(sims, parts):
            keys, grid = _grid(s)
            ranks.append(dict(keys=keys, grid=grid, models=rank_models(ps, [s.particle_state(i) for i in range(len(ps))])))
        dts = [s.stats().dt for s in sims]
        M.check_dts(dts, dts[0], 0)
        t = sims[0].sim_time()
        assert all(s.sim_time() == t for s in sims)
        r = M.substep(cfg, ranks, dts[0], case["dt"], S.engine_time_left(sims[0], case), n_models=nm, collider=ccol, t=np.float32(t), objects=objs)
        on_threads(sims, lambda s: (s.step(1), s.sync()))
        done = k + 1
        for s in sims:
            assert s.stats().error == 0, f"{label}: error bits {s.stats().error} after sub-step {k}"
        after = []
        for s, ps in zip(sims, parts):
            keys, grid = _grid(s)
            after.append(dict(keys=keys, grid=grid, states={p["model"]: s.particle_state(i) for i, p in enumerate(ps)}))
        rep = M.compare(cfg, r, after, COLLIDER_KAPPA, STRESS_ALLOW, f_allow, margin=BRANCH_MARGIN)
        check_report(rep, f"{label} sub-step {k}")
        d = np.asarray([s.stats().dt for s in sims], np.float32)
        assert np.all(d.view(np.int32) == d[0].view(np.int32)), f"{label}: the ranks' dt differ after sub-step {k}: {d}"
        check_dt_range(float(d[0]), r, f"{label} sub-step {k}")
        near += r["near"]
        tainted += rep["tainted_cells"]
    for s in sims:
        s.close()
    print(f"{label}: {near} near nodes, {tainted} tainted cells")
    return r


@pytest.mark.timeout(600)
@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
def test_mgsp_sticky_floor_two_slabs(cuda_lib, use_graph):
    """A CFL-bound block falling onto a sticky floor, cut into two x slabs: the floor resolves the nodes under it."""
    dx = 1.0 / 64
    case = S._case(6, [S.model(S.FIXED_COROTATED, S.box(dx, (24, 20, 24), (36, 28, 34)), (1.0, -10.0, 0.5), dx)], [0, 1, 2, 3, 4], dt=1e-3,
                   collider=dict(field=S.FLOOR, type=S.STICKY, friction=0.3))
    mgsp_collider_check(case, split_case(case, 2, "x"), use_graph, f"sticky floor 2x {'graph' if use_graph else 'stream'}")


@pytest.mark.timeout(600)
@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
def test_mgsp_combined_paddle_2x2(cuda_lib, use_graph):
    """The combined-motion paddle on 2 x 2 ranks: the max comes from nodes the paddle resolves and moves with t, so a predictor
    that placed the collider at any other time than the next grid update's would give another dt.  Sub-step 0 checks the
    set-up predictor (its max is the paddle's object velocity at t = 0)."""
    case = S.COLLIDER_CASES["paddle_combined"]
    r = mgsp_collider_check(case, split_case(case, 4, "2x2"), use_graph, f"paddle 2x2 {'graph' if use_graph else 'stream'}")
    assert r["new_dt"] < case["dt"], "the paddle's dt must be CFL-bound"
