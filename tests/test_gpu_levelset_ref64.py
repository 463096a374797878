"""The step driver and the MGSP dt predictors with level-set collision objects (DESIGN.md section 2.11) against the float64
reference, sub-step by sub-step, with the boundary bounds of ref64_checks (COLLIDER_KAPPA per particle and cell, dt within
DT_ULPS).  ref64's sub-step answers the level-set objects through ref64_levelset.registered.

Step driver: a block falling onto a level-set floor for four materials x three types; a fluid block through the moving,
turning dragonish obstacle (graph and stream); a level-set object after the dense collider and between two analytic objects.
Each runs 40 sub-steps.  MGSP: two x slabs on a rising sticky level-set floor with a CFL-bound dt: after every checked sub-step
both ranks' dt is bit-identical and ref64's; the set-up predictor (grid_max_levelset_kernel) gives sub-step 0's dt and the
carry predictor (carry_grid_levelset_kernel) every later one, so both must apply the level set at the right time.
"""
import numpy as np
import pytest

import ref64_cases as S
import ref64_levelset as RL
from ref64_checks import engine_substep_check, mgsp_substep_check
from test_levelset_objects_cpu import level_set
from test_ref64_mgsp_cpu import split_case

pytestmark = pytest.mark.gpu
DX = 1.0 / 64
STEPS = [0, 5, 20, 39]
FLOOR_LS = level_set("box")          # solid on [0.3, 1.5] x [0.5, 2.1] x [0.35, 1.2] in the file's units
DRAGON_LS = level_set("dragonish")
MATERIALS = {"jfluid": S.J_FLUID, "fixed_corotated": S.FIXED_COROTATED, "sand": S.SAND, "nacc": S.NACC}
TYPES = {"sticky": S.STICKY, "slip": S.SLIP, "separate": S.SEPARATE}


def _lattices(case):
    """the lattices of the case's level sets, in the order the simulator registers them (first use in list order)"""
    seen = []
    for shape, args, _ in case.get("objects", ()):
        if shape == "levelset" and not any(args[0] is s for s in seen):
            seen.append(args[0])
    assert len(seen) <= 1, "ref64_cases' structs carry index 0: one level set per case"
    return [RL.lattice(ls.n, ls.phi) for ls in seen]


def _floor(**kw):
    # the box lattice with node spacing c = 0.5333 / 8 = 0.06667 (z decides the fit): its solid [1.5, 7.5] x [2.5, 10.5] x [1.75, 6]
    # in node units lies at x 0.3-0.7, y -0.17-0.3642 (top off the nodes, just under the blocks' lowest particles at 0.3711), z
    # 0.3283-0.6117, under every block of this file
    return ("levelset", (FLOOR_LS, (0.2, -0.336, 0.2117), (0.61, 0.88, 0.5333)), kw)


def _check(case, use_graph, label):
    with RL.registered(_lattices(case)):
        engine_substep_check(case, use_graph, label)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("typ", list(TYPES))
@pytest.mark.parametrize("material", list(MATERIALS))
def test_block_onto_levelset_floor(cuda_lib, material, typ):
    case = S._case(6, [S.model(MATERIALS[material], S.box(DX, (26, 24, 26), (34, 30, 34)), (0.3, -3.0, 0.2), DX)], STEPS, dt=2e-4,
                   objects=[_floor(type=TYPES[typ], friction=0.3)])
    if material == "sand":   # F = I at sub-step 0: every particle sits on the cone tip (as obj_floor_sand_sticky)
        case["max_near_branch"] = 1.0
    _check(case, True, f"{material} onto a {typ} level-set floor")


@pytest.mark.timeout(900)
@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
def test_fluid_through_moving_turning_dragon(cuda_lib, use_graph):
    # x 0.42-0.51, y 0.42-0.56, z 0.25-0.75 at t = 0: in the block's lower half from the first sub-step
    dragon = ("levelset", (DRAGON_LS, (0.42, 0.42, 0.25), (0.5, 0.5, 0.5)),
              dict(type=S.SLIP, friction=0.2, trans=(0.47, 0.49, 0.5), trans_vel=(0.0, 0.3, 0.1), omega=(0.2, 1.5, -0.4), scale=1.05, dsdt=0.1))
    case = S._case(6, [S.model(S.J_FLUID, S.box(DX, (26, 32, 24), (36, 40, 40)), (0.0, -2.0, 0.0), DX)], STEPS, dt=2e-4, objects=[dragon])
    _check(case, use_graph, f"fluid through the dragon {'graph' if use_graph else 'stream'}")


@pytest.mark.timeout(900)
def test_levelset_with_dense_collider_and_analytic_objects(cuda_lib):
    objs = [("box", ((0.4, 0.36, 0.4), (0.47, 0.42, 0.6)), dict(type=S.SLIP, friction=0.3)), _floor(type=S.SEPARATE, friction=0.3),
            ("sphere", ((0.56, 0.38, 0.5), 0.05), dict(type=S.STICKY))]
    case = S._case(6, [S.model(S.FIXED_COROTATED, S.box(DX, (26, 28, 26), (38, 34, 36)), (0.3, -3.0, 0.2), DX)], STEPS, dt=2e-4,
                   collider=dict(type=S.SLIP, friction=0.0, field=("plane", (0.5, 0.2, 0.5), (0.2, 1.0, 0.0))), objects=objs)
    _check(case, True, "level set with the dense collider and two analytic objects")


@pytest.mark.timeout(900)
@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
def test_mgsp_rising_sticky_levelset_floor_two_slabs(cuda_lib, use_graph):
    # the floor rises at 15 m/s, faster than the block falls: the nodes it holds set the max, so the dt of every sub-step comes
    # from the level set in the predictors
    case = S._case(6, [S.model(S.FIXED_COROTATED, S.box(DX, (24, 24, 24), (36, 30, 34)), (1.0, -3.0, 0.5), DX)], [0, 1, 2, 3, 4],
                   dt=1e-3, objects=[_floor(type=S.STICKY, friction=0.3, trans_vel=(0.0, 15.0, 0.0))])
    with RL.registered(_lattices(case)):
        _, r = mgsp_substep_check(case, split_case(case, 2, "x"), use_graph, f"rising level-set floor 2x {'graph' if use_graph else 'stream'}")
    assert r["new_dt"] < case["dt"], "the dt must be CFL-bound"
