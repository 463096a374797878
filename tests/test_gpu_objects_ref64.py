"""The engine's analytic collision objects against the float64 reference (ref64.object_chain), with the kappa values
test_ref64_objects_cpu.py checks on the FP32 objects oracle (no re-tuning here).

Kernel level: cb200_update_grid_velocity_query_max_objects on the synthetic grids and matrix of the CPU test (every shape, type,
friction, motion, t and boundary, the 16-object list, the level-set collider with two objects), per node and in the max.
Step driver: every case of OBJECT_CASES in graph and stream mode, one sub-step at a time, the objects placed at the simulated
time the engine reports before the sub-step: error bits, the clock, particles and cells, dt.  MGSP: sub-step 0's dt comes
from the set-up predictor (grid_max_boundary_kernel at sim_time), every later one from carry_grid_boundary_kernel, which places
the objects at sim_time + dt; both must be bit-identical on every rank and within DT_ULPS of ref64's grid update at that time.
"""
import ctypes as C

import numpy as np
import pytest

import ref64_cases as S
from ref64_checks import engine_substep_check, mgsp_substep_check
from test_ref64_collider_cpu import FIELDS, block_field
from test_ref64_mgsp_cpu import split_case
from test_ref64_objects_cpu import KERNEL_MATRIX, kernel_matrix

pytestmark = pytest.mark.gpu


# ---- kernel level ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def engine_objects_kernel(cuda_lib):
    """run(cfg, keys, grid, dt, collider spec or None, objects, t) through cb200_update_grid_velocity_query_max_objects"""
    import torch
    from claymore_b200 import objects
    from claymore_b200._capi import Collider, Config, Partition
    cfg0 = Config(domain_bits=6)
    sdf, grad = S.make_field(cfg0.domain_bits, FIELDS["sphere"])
    field = torch.from_numpy(block_field(cfg0.domain_bits, sdf, grad)).cuda()

    def run(cfg, keys, grid, dt, spec, objs, t):
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
        assert cuda_lib.cb200_update_grid_velocity_query_max_objects(C.byref(ecfg), len(keys), C.c_void_p(g.data_ptr()), part, dt,
                                                                     C.byref(col) if col is not None else None, objects.array(objs), len(objs),
                                                                     float(np.float32(t)), C.c_void_p(mv.data_ptr()), None) == 0
        torch.cuda.synchronize()
        return g.cpu().numpy(), float(mv.item())
    return run


@pytest.mark.parametrize("entry,boundary,motion", KERNEL_MATRIX, ids=[f"{e}-b{b}-{m}" for e, b, m in KERNEL_MATRIX])
def test_engine_objects_kernel_matches_ref64(oracle, engine_objects_kernel, entry, boundary, motion):
    worst, near, total, _ = kernel_matrix(engine_objects_kernel, oracle, entry, boundary, motion, f"cb200 {entry} boundary {boundary} {motion}")
    print(f"cb200 {entry} boundary {boundary} {motion}: worst {worst:.3f} x COLLIDER_VEL_KAPPA, {near} of {total} nodes near")


# ---- step driver ----------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(600)
@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
@pytest.mark.parametrize("name", list(S.OBJECT_CASES))
def test_engine_object_substep_matches_ref64(cuda_lib, name, use_graph):
    engine_substep_check(S.OBJECT_CASES[name], use_graph, f"{name} {'graph' if use_graph else 'stream'}")


# ---- MGSP -------------------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(600)
@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
def test_mgsp_analytic_sticky_floor_two_slabs(cuda_lib, use_graph):
    """A CFL-bound block falling onto a sticky analytic floor, cut into two x slabs."""
    dx = 1.0 / 64
    case = S._case(6, [S.model(S.FIXED_COROTATED, S.box(dx, (24, 20, 24), (36, 28, 34)), (1.0, -10.0, 0.5), dx)], [0, 1, 2, 3, 4], dt=1e-3,
                   objects=[("box", (S.FLOOR_LO, S.FLOOR_HI), dict(type=S.STICKY, friction=0.3))])
    mgsp_substep_check(case, split_case(case, 2, "x"), use_graph, f"analytic sticky floor 2x {'graph' if use_graph else 'stream'}")


@pytest.mark.timeout(600)
@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
def test_mgsp_object_paddle_2x2(cuda_lib, use_graph):
    """The combined-motion paddle object on 2 x 2 ranks: the max comes from nodes the paddle resolves and moves with t, so a
    predictor that placed the objects at any other time than the next grid update's would give another dt."""
    case = S.OBJECT_CASES["obj_paddle_combined"]
    _, r = mgsp_substep_check(case, split_case(case, 4, "2x2"), use_graph, f"object paddle 2x2 {'graph' if use_graph else 'stream'}")
    assert r["new_dt"] < case["dt"], "the paddle's dt must be CFL-bound"


@pytest.mark.timeout(600)
def test_mgsp_collider_plus_objects_two_slabs(cuda_lib):
    """The level-set collider with two objects on two x slabs: the <true> forms of both predictors."""
    case = S.OBJECT_CASES["obj_collider_plus_two"]
    mgsp_substep_check(case, split_case(case, 2, "x"), True, "collider + objects 2x graph")
