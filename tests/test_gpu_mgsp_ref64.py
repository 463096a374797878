"""MGSP ranks against the float64 reference (tests/ref64_mgsp.py), per grid copy and per particle, with the kappa values the FP32
oracle fixed (test_ref64_cpu.py, test_ref64_mgsp_cpu.py; no re-tuning here).

All ranks of a case live in this process on one GPU, peers wired with mgsp_set_peers; every rank's initial_setup and step
runs on a host thread of its own (the ranks' exchange kernels wait for each other), in graph and stream mode.  One sub-step
at a time: every rank's state at sub-step k, one sub-step on every rank, then every rank's copy of every block, the union of
the ranks' particles per scene model and every rank's dt against the reference.  At most 4 ranks: the exchange kernels of
every rank spin on their peers' flags, and more ranks on one GPU could leave no SM for the last rank's wide kernels.
"""
import pytest

import ref64_cases as S
from ref64_checks import ERR_BLOCK_CAPACITY, build_ranks, mgsp_substep_check
from test_ref64_mgsp_cpu import split_case

pytestmark = pytest.mark.gpu


CROSSING = 0.25 / 64 / (2.5 * 1e-4)   # m/s: carries a lattice particle (0.25 dx short of a cell face) across it in sub-step 3


def _slabs_into_each_other():
    """Two fixed-corotated slabs on either side of the cut driven towards each other (x velocity +-CROSSING, the same transverse
    drift): slab A's front cell is the last of its particle block and slab B's back cell the first of its, so at sub-step 3 each
    rank's partition grows into a block the other rank already holds (a fresh copy on both ranks), and again at later crossings.
    (A drift is kept on the transverse axes: with a purely axis-aligned velocity the FP32 oracle leaves ref64's F bound on
    the off-diagonal entries, whose magnitude is then only the gravity term.)"""
    dx = 1.0 / 64
    return S._case(6, [S.model(S.FIXED_COROTATED, S.box(dx, (12, 20, 20), (22, 32, 32)), (CROSSING, -1.5, 1.0), dx),
                       S.model(S.FIXED_COROTATED, S.box(dx, (26, 20, 20), (36, 32, 32)), (-CROSSING, -1.5, 1.0), dx)], list(range(10)))


def _cfl_two_speeds():
    """A CFL-bound pair of cubes on two ranks: rank 1's cube is ten times faster, so the global max |v|^2 (and dt) is rank 1's,
    and a rank that kept its own maximum would pick a different dt."""
    dx = 1.0 / 64
    return S._case(6, [S.model(S.FIXED_COROTATED, S.box(dx, (20, 20, 20), (26, 26, 26)), (0.3, -1.0, 0.2), dx),
                       S.model(S.FIXED_COROTATED, S.box(dx, (28, 20, 20), (34, 26, 26)), (1.0, -10.0, 0.5), dx)], [0, 1, 2, 3], dt=1e-3)


def _high_faces_by_group():
    """high_faces with each of its four groups (x, y, z top faces and the top corner, 64 particles each) as a model of its own,
    so that cutting every model in x shares the blocks at the top faces."""
    c = S.CASES["high_faces"]
    m = c["models"][0]
    return dict(c, models=[dict(m, pos=m["pos"][64 * i: 64 * (i + 1)]) for i in range(4)])


def _movers():
    """A lattice cube crossing cell faces at sub-step 3 (test_gpu_movers' crossing velocity), cut in x at the last cell of a particle
    block: rank 0's front particles enter a particle block whose neighbour rank 1 already holds (fresh copies on rank 0)."""
    dx = 1.0 / 64
    return S._case(6, [S.model(S.FIXED_COROTATED, S.box(dx, (20, 20, 20), (32, 32, 32)), (CROSSING, -1.5, 1.0), dx)], list(range(8)))


# name -> (case, world, split, what the run must show)
MATRIX = {
    "fc_cube-2x": (S.CASES["fc_cube"], 2, "x", dict(owners=2)),
    "fc_cube-3x": (S.CASES["fc_cube"], 3, "x", dict(owners=3)),
    "fc_cube-2x2": (S.CASES["fc_cube"], 4, "2x2", dict(owners=4)),
    "fluid_cube-2x": (S.CASES["fluid_cube"], 2, "x", dict(owners=2)),
    "nacc_cube-2x": (S.CASES["nacc_cube"], 2, "x", dict(owners=2)),
    "cfl_bound-2x": (S.CASES["cfl_bound"], 2, "x", dict(owners=2)),
    "cfl_bound-2x2": (S.CASES["cfl_bound"], 4, "2x2", dict(owners=4)),
    "cfl_two_speeds-2global": (_cfl_two_speeds(), 2, "global", dict(owners=2)),
    "fc_floor_frame_end-2x": (S.CASES["fc_floor_frame_end"], 2, "x", dict(owners=2)),
    "walls-2x": (S.CASES["walls"], 2, "x", dict(owners=2)),
    "high_faces-2x": (_high_faces_by_group(), 2, "x", dict(owners=2)),
    "multi_model_8-2global": (S.CASES["multi_model_8"], 2, "global", dict(owners=2, models_differ=True)),
    # rho changes between sub-steps on the ranks that hold the model (ref64_checks.rank_update); a rank without it makes no call
    "multi_model_8_params-2global": (S.CASES["multi_model_8_params"], 2, "global", dict(owners=2, models_differ=True)),
    "block_sizes-2x": (S.CASES["block_sizes"], 2, "x", dict(owners=2, models_differ=True)),
    "slabs_into_each_other-2global": (_slabs_into_each_other(), 2, "global", dict(owners=2, fresh=True)),
    "movers-2x": (_movers(), 2, "x", dict(owners=2, fresh=True)),
}


@pytest.mark.timeout(600)
@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
@pytest.mark.parametrize("name", list(MATRIX))
def test_mgsp_ranks_match_ref64(cuda_lib, name, use_graph):
    case, world, kind, want = MATRIX[name]
    parts = split_case(case, world, kind)
    lists = [sorted(p["model"] for p in ps) for ps in parts]
    if want.get("models_differ"):
        assert any(a != b for a in lists for b in lists), lists   # a rank holds a model another rank lacks
    seen, _ = mgsp_substep_check(case, parts, use_graph, f"{name} {'graph' if use_graph else 'stream'}")
    print(f"{name}: {seen}, model lists {lists}")
    assert seen["max_owners"] >= want["owners"], seen
    if want.get("fresh"):   # zero copies seen after a sub-step, then filled from their owners in the next sub-step's input
        assert seen["fresh"] > 0 and seen["fresh_in"] > 0, seen


@pytest.mark.timeout(300)
def test_mgsp_halo_capacity_at_setup(cuda_lib):
    """mgsp_halo_cap equal to the largest per-peer overlap count at set-up sets no error bit; one less sets kErrBlockCapacity on
    exactly the ranks whose overlap with some peer exceeds it."""
    case = S.CASES["fc_cube"]
    parts = split_case(case, 3, "x")
    sims = build_ranks(case, parts, True)
    counts = [s.mgsp_halo_counts()[0] for s in sims]
    for s in sims:
        s.close()
    cap = max(max(c) for c in counts)
    assert cap > 0
    for halo_cap, want in ((cap, [0] * 3), (cap - 1, [ERR_BLOCK_CAPACITY if max(c) > cap - 1 else 0 for c in counts])):
        sims = build_ranks(case, parts, True, halo_cap=halo_cap)
        got = [s.stats().error & ERR_BLOCK_CAPACITY for s in sims]
        assert got == want, (halo_cap, counts, got)
        for s in sims:
            s.close()
