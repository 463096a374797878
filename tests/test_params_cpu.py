"""The power of the parameter-change cases of ref64_cases (case["updates"]): each would catch a runner that kept a stale parameter.

For every update of every such case, the FP32 oracle is run to the update's sub-step k with every update before it applied, the
update is applied, and the oracle's sub-step k is compared with ref64 twice, with the bounds ref64_checks holds every runner to:
with the parameters after the update it must pass; with that model's parameters before the update it must fail, by at least
POWER times the bound on some grid cell or particle.  Updates of one sub-step are undone one model at a time.
"""
import numpy as np
import pytest

import ref64
import ref64_cases as S
from ref64_checks import BRANCH_MARGIN, F_ALLOW, KAPPA, STRESS_ALLOW, apply_updates, check_report, current_models, ref_models

POWER = 10.0
UPDATE_CASES = [n for n, c in S.CASES.items() if c.get("updates")]


def test_update_cases_cover_every_setter_and_both_parities():
    materials = {S.CASES[n]["models"][mi]["material"] for n in UPDATE_CASES for ups in S.CASES[n]["updates"].values() for mi, *_ in ups}
    assert materials == {S.J_FLUID, S.FIXED_COROTATED, S.SAND, S.NACC}
    ks = [k for n in UPDATE_CASES for k in S.CASES[n]["updates"]]
    assert min(ks) >= 1 and {k % 2 for k in ks} == {0, 1}


@pytest.mark.parametrize("name", UPDATE_CASES)
def test_stale_parameters_fail_the_bounds(oracle, name):
    case = S.CASES[name]
    nm = len(case["models"])
    osim = S.build_oracle(oracle, case)
    clock = S.OracleClock(osim)
    models = current_models(case)
    done = 0
    for k in sorted(case["updates"]):
        clock.step(k - done)
        old = [dict(m) for m in models]
        apply_updates(case, k, models, lambda mi, setter, rho, vol, args: getattr(osim, setter)(mi, rho, vol, *args))
        _, nbc, _ = osim.block_counts()
        keys, grid = osim.active_keys()[:nbc], osim.grid()
        before = [osim.particle_state(i) for i in range(nm)]
        stale = {}
        for mi, *_ in case["updates"][k]:
            ms = [dict(m) for m in models]
            ms[mi] = old[mi]
            stale[mi] = ms
        runs = [("new", models)] + [(f"model {mi} before the update", ms) for mi, ms in stale.items()]
        refs = [(label, ref64.substep(osim.cfg, ref_models(case, before, ms), keys, grid, osim.dt, case["dt"], clock.time_left())) for label, ms in runs]
        clock.step(1)
        done = k + 1
        _, nbc, _ = osim.block_counts()
        after = [osim.particle_state(i) for i in range(nm)]
        for label, r in refs:
            rep = ref64.compare(r, osim.active_keys()[:nbc], osim.grid(), after, KAPPA, STRESS_ALLOW, [F_ALLOW[m["material"]] for m in case["models"]],
                                margin=BRANCH_MARGIN, max_ppc=case["max_ppc"])
            if label == "new":
                check_report(rep, f"{name} sub-step {k}")
            else:
                worst = max(rep[q] for q in ("mass", "momentum", "pos", "F"))
                assert worst >= POWER, f"{name} sub-step {k}, {label}: the oracle is within {worst:.3g} x the bound ({rep})"
    osim.close()
