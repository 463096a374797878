"""The sub-step checks against the float64 reference (tests/ref64.py, ref64_mgsp.py): one loop per runner, the FP32 oracle, the
step driver and in-process MGSP ranks, and the bounds they hold each sub-step to.

Every loop runs a case of ref64_cases through case['steps']: the runner's state at sub-step k -> ref64 for one sub-step ->
compared with the runner at k + 1 per grid cell (by key) and per particle (matched by position), each against its own bound
kappa * 2^-24 * M (ref64.compare), then the dt.  The bounds come from the case (boundary_bounds): a case with a collider or
collision objects gets COLLIDER_KAPPA, the dt within the range of the near nodes' branch choices (check_dt_range) and caps on the
near nodes and the particles that read them (collider_report); any other case gets KAPPA and the dt within DT_ULPS (check_dt).
The kappa values are the smallest round values the FP32 oracle passes over the matrices of test_ref64_cpu.py and
test_ref64_collider_cpu.py; the GPU tests hold the engine to the same values.
"""
import threading

import numpy as np

import ref64
import ref64_cases as S
import ref64_mgsp as M

# kappa per quantity; beside each, the oracle's worst |oracle - ref64| / (2^-24 M) over ref64_cases.CASES
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

# the collider's grid velocity per component: the oracle's worst |oracle - ref64| / (2^-24 E) over test_ref64_collider_cpu's
# KERNEL_MATRIX is 2.62 (box, boundary 0, static), against 2.13 for the grid update without a collider (VEL_KAPPA 4 there, as here)
COLLIDER_VEL_KAPPA = 4.0
MAX_NEAR_NODES = 0.01      # share of the resolved nodes that may lie near a discontinuity
MAX_TAINTED = 0.05         # share of the particle updates (and of the grid cells) that may read (write) such a node
# Per sub-step with boundaries: KAPPA, except F (J, F, logJp): 8 in place of 4.  The oracle's worst F is 5.9 on
# walls_boundary1, which has no collider: a wall band's edge runs through its models, so the grid velocity jumps from v to 0
# between two nodes, and F's M has no term for the last bit of the stored position (the momentum's has one) while G2P's
# weights carry that bit times |v| / dx into A.  The collider cases stay under 4.6 (moving_floor_frame_end, sphere_separate).
COLLIDER_KAPPA = dict(KAPPA, F=8.0)

# the engine's error bits (kErrBlockCapacity, kErrLost, kErrCellOverflow, kErrHaloMap)
ERR_BLOCK_CAPACITY, ERR_LOST, ERR_CELL_OVERFLOW, ERR_HALO_MAP = 1, 4, 8, 16


def boundary_bounds(case):
    """Whether the case is held to the boundary bounds: it has a collider or collision objects, or asks for them."""
    return bool(case.get("collider") or case.get("objects") or case.get("boundary_bounds"))


# ---- the pieces of a sub-step check ----------------------------------------------------------------------------------------
def check_report(rep, label):
    for q in ("mass", "momentum", "pos", "F"):
        assert rep[q] <= 1.0, f"{label}: {q} error is {rep[q]:.3g} x its bound ({rep['worst']})"


def check_dt(impl_dt, ref_dt, label):
    ulp = float(np.spacing(np.float32(ref_dt)))
    assert abs(impl_dt - ref_dt) <= DT_ULPS * ulp, f"{label}: dt {impl_dt!r} vs reference {ref_dt!r} ({(impl_dt - ref_dt) / ulp:.2f} ulp)"


def check_dt_range(impl_dt, r, label):
    """The implementation's dt lies in [dt(mx_hi), dt(mx_lo)] (the near nodes' branch choices) within DT_ULPS, the max
    widened by COLLIDER_VEL_KAPPA 2^-24 mx_err (dt scales as max^-1/2 where it is CFL-bound)."""
    lo, hi = r["dt_range"]
    info = r.get("collider_info", r)
    err = COLLIDER_VEL_KAPPA * ref64.EPS32 * info.get("mx_err", 0.0)
    if info["mx_hi"] > 0 and err > 0:
        lo *= np.sqrt(info["mx_hi"] / (info["mx_hi"] + err))
        hi *= np.sqrt(info["mx_lo"] / max(info["mx_lo"] - err, info["mx_lo"] * 0.5)) if info["mx_lo"] > 0 else 1.0
    ulp = float(np.spacing(np.float32(r["new_dt"])))
    assert lo - DT_ULPS * ulp <= impl_dt <= hi + DT_ULPS * ulp, f"{label}: dt {impl_dt!r} outside [{lo!r}, {hi!r}] (ref64 {r['new_dt']!r})"


def check_new_dt(case, impl_dt, r, label):
    if boundary_bounds(case):
        check_dt_range(impl_dt, r, label)
    else:
        check_dt(impl_dt, r["new_dt"], label)


def check_counts(r, before, after, max_ppc, label):
    """No particle disappears unless ref64 says so: the count after a sub-step is n - lost - what overflowing cells drop."""
    for m, (res, b, a) in enumerate(zip(r["models"], before, after)):
        _, n_over, kept = ref64.cell_overflow(res, max_ppc)
        lost = int(res["lost"].sum())
        assert len(a) == kept, (f"{label}: model {m} has {len(a)} particles after the sub-step, {len(b)} before; ref64 predicts {kept} "
                                f"({lost} lost, {len(b) - lost - kept} dropped from {n_over} cells over max_ppc = {max_ppc})")


def ref_models(case, states, models=None):
    """ref64's models of the case's particle ``states``, with the parameters of ``models`` (current_models) or else the case's."""
    return [dict(material=m["material"], params=S.ref_params(m), state=s) for m, s in zip(case["models"] if models is None else models, states)]


def rank_models(parts, states, models=None):
    """ref64_mgsp's models of a rank's ``parts``, with the parameters of the scene models ``models`` (current_models) or else the parts'."""
    return [dict(model=p["model"], material=p["material"], params=S.ref_params(p if models is None else models[p["model"]]), state=s)
            for p, s in zip(parts, states)]


# ---- parameter changes between sub-steps (case["updates"], ref64_cases) -------------------------------------------------------
def current_models(case):
    """The case's models as set up; apply_updates keeps their rho, vol and args at the parameters in effect."""
    return [dict(m) for m in case["models"]]


def apply_updates(case, k, models, call):
    """The case's updates before sub-step k: call(scene model, material setter name, rho, vol, args) for each, and ``models``
    (current_models) follows.  Every update step k and k + 1 must be checked steps: the two roll parities read the parameters of
    pb[0] and pb[1] in turn."""
    for mi, rho, vol, args in case.get("updates", {}).get(k, ()):
        assert k >= 1 and k in case["steps"] and k + 1 in case["steps"], f"an update at sub-step {k} needs sub-steps {k} and {k + 1} checked"
        m = models[mi]
        call(mi, S.SETTER[m["material"]], rho, vol, tuple(args))
        m.update(rho=rho, vol=vol, args=tuple(args))


def new_counts():
    return dict(near=0, resolved=0, tainted_particles=0, tainted_cells=0, near_branch=0, worst={})


def substep_compare(case, r, keys, grid, before, after, dt_after, label, counts):
    """One sub-step of one runner against ref64's ``r`` with the case's bounds; adds to ``counts`` (new_counts)."""
    kappa = COLLIDER_KAPPA if boundary_bounds(case) else KAPPA
    check_counts(r, before, after, case["max_ppc"], label)
    rep = ref64.compare(r, keys, grid, after, kappa, STRESS_ALLOW, [F_ALLOW[m["material"]] for m in case["models"]], margin=BRANCH_MARGIN,
                        max_ppc=case["max_ppc"])
    check_report(rep, label)
    check_new_dt(case, dt_after, r, label)
    info = r["collider_info"]
    if info["near"] is not None:
        counts["near"] += int(info["near"].sum())
        counts["resolved"] += int((info["branch"] != "").sum())   # nodes with mass: the ones the collider resolves
    for q in ("tainted_particles", "tainted_cells", "near_branch"):
        counts[q] += rep[q]
    for q in ("mass", "momentum", "pos", "F"):
        counts["worst"][q] = round(max(counts["worst"].get(q, 0.0), rep[q] * kappa[q] / KAPPA[q]), 3)


def collider_report(case, label, counts):
    """The caps over the whole run: particle updates near a branch point; with boundaries (printed) also near nodes and tainted
    particles."""
    total = sum(len(m["pos"]) for m in case["models"]) * len(case["steps"])
    if boundary_bounds(case):
        print(f"{label}: near nodes {counts['near']} of {counts['resolved']}, tainted particles {counts['tainted_particles']} of {total}, "
              f"tainted cells {counts['tainted_cells']}, worst x KAPPA {counts['worst']}")
        assert counts["near"] <= case.get("max_near_nodes", MAX_NEAR_NODES) * max(counts["resolved"], 1), f"{label}: {counts}"
        assert counts["tainted_particles"] <= case.get("max_tainted", MAX_TAINTED) * total, f"{label}: {counts}"
    # the branch-point exclusion is for the odd particle; a case where it hides a large share proves nothing
    assert counts["near_branch"] <= case.get("max_near_branch", 0.01) * total, f"{label}: {counts['near_branch']} of {total} particle updates near a branch point"


def engine_state(sim, nm):
    g = sim.grid()
    return sim.active_keys()[: len(g)], g, [sim.particle_state(i) for i in range(nm)]


def rank_grid(sim):
    g = sim.grid()
    return sim.active_keys()[: len(g)].astype(np.int64), g


# ---- the loops ---------------------------------------------------------------------------------------------------------------
def oracle_substep_check(ob, case, label):
    """Run the oracle through case['steps']; at each, one ref64 sub-step against the oracle's next one."""
    osim = S.build_oracle(ob, case)
    clock = S.OracleClock(osim)
    ccol, objs = S.ref_collider(case), S.ref_objects(case)
    nm = len(case["models"])
    done = 0
    counts = new_counts()
    models = current_models(case)
    for k in case["steps"]:
        clock.step(k - done)
        apply_updates(case, k, models, lambda mi, setter, rho, vol, args: getattr(osim, setter)(mi, rho, vol, *args))
        t = np.float32(osim.sim_time) if ccol is not None or objs else 0.0
        _, nbc, _ = osim.block_counts()
        before = [osim.particle_state(i) for i in range(nm)]
        r = ref64.substep(osim.cfg, ref_models(case, before, models), osim.active_keys()[:nbc], osim.grid(), osim.dt, case["dt"], clock.time_left(), ccol, t,
                          objects=objs)
        clock.step(1)
        done = k + 1
        _, nbc, _ = osim.block_counts()
        after = [osim.particle_state(i) for i in range(nm)]
        substep_compare(case, r, osim.active_keys()[:nbc], osim.grid(), before, after, osim.dt, f"{label} sub-step {k}", counts)
    osim.close()
    collider_report(case, label, counts)


def engine_substep_check(case, use_graph, label, sim=None, before_step=None, start=0):
    """The step driver through case['steps'], the boundaries placed at the simulated time the engine reports before each
    checked sub-step: error bits, the clock, particles and cells, dt.  ``sim``: a simulator of the case, set up, at sub-step ``start``
    (default: S.build_engine, at 0); ``before_step(sim, k)`` runs after the updates of each checked sub-step k, right before the state is read."""
    sim = S.build_engine(case, use_graph=use_graph) if sim is None else sim
    ccol, objs = S.ref_collider(case), S.ref_objects(case)
    nm = len(case["models"])
    done = start
    expect = 0   # a particle that moves more than one cell (quirk #4) or leaves its block's neighbourhood is flagged lost,
    #              a cell that gets more than max_ppc particles in g2p2g sets the overflow bit
    counts = new_counts()
    models = current_models(case)
    for k in case["steps"]:
        sim.step(k - done)
        apply_updates(case, k, models, lambda mi, setter, rho, vol, args: getattr(sim, setter)(rho, vol, *args, model=mi))
        if before_step is not None:
            before_step(sim, k)
        st = sim.stats()
        assert st.error == expect, f"{label}: error bits {st.error} at sub-step {k}, expected {expect}"
        keys, grid, before = engine_state(sim, nm)
        t = sim.sim_time()
        r = ref64.substep(sim.cfg, ref_models(case, before, models), keys, grid, st.dt, case["dt"], S.engine_time_left(sim, case), ccol, np.float32(t),
                          objects=objs)
        sim.step(1)
        done = k + 1
        assert sim.sim_time() == t + float(np.float32(st.dt)), f"{label}: sim_time {sim.sim_time()!r} after a sub-step of {st.dt!r} from {t!r}"
        st = sim.stats()
        if any(m["dropped"].any() or m["lost"].any() for m in r["models"]):
            expect |= ERR_LOST
        if any(ref64.cell_overflow(m, case["max_ppc"])[1] for m in r["models"]):
            expect |= ERR_CELL_OVERFLOW
        assert st.error == expect, f"{label}: error bits {st.error} after sub-step {k}, expected {expect}"
        keys, grid, states = engine_state(sim, nm)
        substep_compare(case, r, keys, grid, before, states, st.dt, f"{label} sub-step {k}", counts)
    sim.close()
    collider_report(case, label, counts)


def on_threads(sims, fn, timeout=120):
    """fn(sim) for every rank, each on a host thread of its own (the ranks' exchange kernels wait for each other)."""
    errs = []

    def go(s):
        try:
            fn(s)
        except Exception as e:  # pragma: no cover
            errs.append(e)
    th = [threading.Thread(target=go, args=(s,)) for s in sims]
    [t.start() for t in th]
    [t.join(timeout) for t in th]
    assert not errs and not any(t.is_alive() for t in th), errs


def build_ranks(case, parts, use_graph, halo_cap=0, max_blocks=6000):
    """In-process MGSP ranks of ``parts`` (test_ref64_mgsp_cpu.split_case), peers wired, with the case's collider and objects set
    before initial_setup, so that the set-up's next-max predictor (grid_max_boundary_kernel) applies them."""
    from claymore_b200.simulator import GmpmSimulator
    sims = []
    for r, ps in enumerate(parts):
        sim = GmpmSimulator(dt=case["dt"], fps=case.get("fps", 0), config=S.config(case), max_blocks=max_blocks, use_graph=use_graph,
                            mgsp_rank=r, mgsp_world=len(parts), mgsp_halo_cap=halo_cap)
        for p in ps:
            mid = sim.init_model(p["material"], p["pos"], p["v0"])
            getattr(sim, S.SETTER[p["material"]])(p["rho"], p["vol"], *p["args"], model=mid)
        S.set_boundaries(sim, case)
        sims.append(sim)
    ptrs = [s.mgsp_inbox() for s in sims]
    for s in sims:
        s.mgsp_set_peers(ptrs)
    on_threads(sims, lambda s: s.initial_setup())
    return sims


def rank_update(sims, parts, mi, setter, rho, vol, args):
    """A parameter change of scene model ``mi`` on every rank that holds it (its local model id is its index in the rank's parts)."""
    for s, ps in zip(sims, parts):
        for i, p in enumerate(ps):
            if p["model"] == mi:
                getattr(s, setter)(rho, vol, *args, model=i)


def rank_errors(sims, expect, label):
    got = [s.stats().error for s in sims]
    assert not any(e & ERR_HALO_MAP for e in got), f"{label}: kErrHaloMap on a rank ({got})"
    assert got == expect, f"{label}: error bits {got}, expected {expect}"


def mgsp_substep_check(case, parts, use_graph, label):
    """Set-up grid and case['steps'] sub-steps of the ranks against ref64_mgsp, the boundaries at the engine's sim_time: every
    rank's copy of every block, the union of the ranks' particles per scene model, every rank's error bits and dt (bit-identical
    on every rank; sub-step 0's from the set-up predictor, every later one from the carry kernel's).  Returns what the ranks saw
    (owners, fresh copies) and the reference of the last sub-step."""
    sims = build_ranks(case, parts, use_graph)
    cfg = sims[0].cfg
    ccol, objs = S.ref_collider(case), S.ref_objects(case)
    kappa = COLLIDER_KAPPA if boundary_bounds(case) else KAPPA
    nm = len(case["models"])
    seen = dict(max_owners=0, fresh=0, fresh_in=0)
    expect = [0] * len(sims)
    rank_errors(sims, expect, f"{label} set-up")
    ref = M.rasterize(cfg, [[dict(pos=p["pos"], v0=p["v0"], mass=S.ref_params(p)["mass"]) for p in ps] for ps in parts])
    check_report(M.compare(cfg, ref, [dict(zip(("keys", "grid"), rank_grid(s))) for s in sims], RASTER_KAPPA, 0.0, []), f"{label} set-up")
    done, near_branch, near, tainted = 0, 0, 0, 0
    f_allow = [F_ALLOW[m["material"]] for m in case["models"]]
    models = current_models(case)
    for k in case["steps"]:
        if k > done:
            on_threads(sims, lambda s: (s.step(k - done), s.sync()))
        apply_updates(case, k, models, lambda mi, setter, rho, vol, args: rank_update(sims, parts, mi, setter, rho, vol, args))
        rank_errors(sims, expect, f"{label} at sub-step {k}")
        ranks = []
        for s, ps in zip(sims, parts):
            keys, grid = rank_grid(s)
            ranks.append(dict(keys=keys, grid=grid, models=rank_models(ps, [s.particle_state(i) for i in range(len(ps))], models)))
        dts = [s.stats().dt for s in sims]
        M.check_dts(dts, dts[0], 0)
        t = sims[0].sim_time()
        assert all(s.sim_time() == t for s in sims)
        r = M.substep(cfg, ranks, dts[0], case["dt"], S.engine_time_left(sims[0], case), n_models=nm, collider=ccol, t=np.float32(t), objects=objs)
        on_threads(sims, lambda s: (s.step(1), s.sync()))
        done = k + 1
        for i, per in enumerate(r["per_rank"]):
            if any(res["dropped"].any() or res["lost"].any() for _, res in per):
                expect[i] |= ERR_LOST
        rank_errors(sims, expect, f"{label} after sub-step {k}")
        after = []
        for s, ps in zip(sims, parts):
            keys, grid = rank_grid(s)
            after.append(dict(keys=keys, grid=grid, states={p["model"]: s.particle_state(i) for i, p in enumerate(ps)}))
        rep = M.compare(cfg, r, after, kappa, STRESS_ALLOW, f_allow, margin=BRANCH_MARGIN)
        check_report(rep, f"{label} sub-step {k}")
        dts = [s.stats().dt for s in sims]
        M.check_dts(dts, dts[0], 0)
        check_new_dt(case, float(np.float32(dts[0])), r, f"{label} sub-step {k}")
        near_branch += rep["near_branch"]
        near += r["near"]
        tainted += rep["tainted_cells"]
        seen["max_owners"] = max(seen["max_owners"], rep["max_owners"])
        seen["fresh"] += rep["fresh"]
        seen["fresh_in"] += r["fresh_in"]
    for s in sims:
        s.close()
    if boundary_bounds(case):
        print(f"{label}: {near} near nodes, {tainted} tainted cells")
    total = sum(len(m["pos"]) for m in case["models"]) * len(case["steps"])
    assert near_branch <= case.get("max_near_branch", 0.01) * total, f"{label}: {near_branch} of {total} particle updates near a branch point"
    return seen, r
