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

import ref64_cases as S
from ref64_checks import engine_substep_check, mgsp_substep_check
from test_ref64_collider_cpu import FIELDS, KERNEL_MATRIX, block_field, kernel_matrix
from test_ref64_mgsp_cpu import split_case

pytestmark = pytest.mark.gpu


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
@pytest.mark.timeout(600)
@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
@pytest.mark.parametrize("name", list(S.COLLIDER_CASES))
def test_engine_collider_substep_matches_ref64(cuda_lib, name, use_graph):
    engine_substep_check(S.COLLIDER_CASES[name], use_graph, f"{name} {'graph' if use_graph else 'stream'}")


# ---- MGSP -------------------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(600)
@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
def test_mgsp_sticky_floor_two_slabs(cuda_lib, use_graph):
    """A CFL-bound block falling onto a sticky floor, cut into two x slabs: the floor resolves the nodes under it."""
    dx = 1.0 / 64
    case = S._case(6, [S.model(S.FIXED_COROTATED, S.box(dx, (24, 20, 24), (36, 28, 34)), (1.0, -10.0, 0.5), dx)], [0, 1, 2, 3, 4], dt=1e-3,
                   collider=dict(field=S.FLOOR, type=S.STICKY, friction=0.3))
    mgsp_substep_check(case, split_case(case, 2, "x"), use_graph, f"sticky floor 2x {'graph' if use_graph else 'stream'}")


@pytest.mark.timeout(600)
@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
def test_mgsp_combined_paddle_2x2(cuda_lib, use_graph):
    """The combined-motion paddle on 2 x 2 ranks: the max comes from nodes the paddle resolves and moves with t, so a predictor
    that placed the collider at any other time than the next grid update's would give another dt.  Sub-step 0 checks the
    set-up predictor (its max is the paddle's object velocity at t = 0)."""
    case = S.COLLIDER_CASES["paddle_combined"]
    _, r = mgsp_substep_check(case, split_case(case, 4, "2x2"), use_graph, f"paddle 2x2 {'graph' if use_graph else 'stream'}")
    assert r["new_dt"] < case["dt"], "the paddle's dt must be CFL-bound"
