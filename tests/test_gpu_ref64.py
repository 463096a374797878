"""The engine's sub-step against the float64 reference (tests/ref64.py), per grid cell and per particle, with the kappa
values the FP32 oracle fixed (ref64_checks, test_ref64_cpu.py; no re-tuning here), and the engine's set-up rules at the domain's
faces and limits.

The step driver is the production path (the sorted g2p2g with arrival lists), in graph and stream mode: the engine's
particle_state, grid(), active_keys() and stats().dt at sub-step k, one sub-step, then the engine at k + 1 against ref64
applied to the state at k.
"""
import ctypes as C

import numpy as np
import pytest

import ref64
import ref64_cases as S
from ref64_checks import ERR_CELL_OVERFLOW, ERR_LOST, RASTER_KAPPA, check_report, engine_substep_check
from test_ref64_cpu import KERNEL_LEVEL, KERNEL_LEVEL_CASES, grid_mass, kernel_level_check

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
@pytest.mark.parametrize("name", list(S.CASES))
def test_engine_substep_matches_ref64(cuda_lib, name, use_graph):
    engine_substep_check(S.CASES[name], use_graph, name)


@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
def test_engine_substep_matches_ref64_when_a_lattice_crosses_a_face(cuda_lib, use_graph):
    """test_gpu_movers' velocities: the particle sub-lattice crosses a cell face in the checked sub-steps (movers inside and
    out of the particle block, arrival lists)."""
    dx = 1.0 / 64
    for v0 in ((2.5, 0.0, 0.0), (2.0, -1.5, 1.0)):
        case = S._case(6, [S.model(S.FIXED_COROTATED, S.box(dx, (20, 20, 20), (32, 32, 32)), v0, dx)], [0, 4, 8, 12])
        engine_substep_check(case, use_graph, f"movers {v0}")


@pytest.mark.parametrize("name", ["overflow_fc_in_block", "overflow_fluid_cross_block"])
def test_cell_overflow_in_g2p2g_engine(cuda_lib, name):
    """A cell that receives more than max_ppc particles in g2p2g: kErrCellOverflow, the cell keeps max_ppc of them; the grid of
    that sub-step has every particle's mass, the next one is short by exactly the mass of the dropped particles (the per-cell
    and per-particle rules are engine_substep_check's, through the case in the matrix)."""
    case = S.CASES[name]
    sim = S.build_engine(case)
    n = len(case["models"][0]["pos"])
    mass = S.ref_params(case["models"][0])["mass"]
    sim.step(1)
    assert sim.stats().error == ERR_CELL_OVERFLOW, sim.stats().error
    assert len(sim.particle_state(0)) == n - 9 * 4
    assert abs(grid_mass(sim.grid()) - n * mass) <= 1e-6 * n * mass
    sim.step(1)
    assert abs(grid_mass(sim.grid()) - (n - 9 * 4) * mass) <= 1e-6 * n * mass
    sim.close()


# ---- set-up rules at the faces and limits -------------------------------------------------------------------------------
def test_low_face_rule_step_driver_floors_and_flags_lost(cuda_lib):
    """A particle less than 1.5 dx from a low face (cell index 0 or 1: cell - 2 < 0) has a negative particle block under floor
    semantics, the rule g2p2g's stencil and re-bucketing use.  The step driver flags it lost at set-up and does not bucket it;
    particles at cell index 2 (and at the top face, 4G - 1 and 4G) are kept."""
    dx = 1.0 / 64
    inner = S.box(dx, (20, 20, 20), (24, 24, 24))
    edge = np.array([[0.2, 30.1, 30.1], [1.1, 30.1, 30.1], [30.1, 0.9, 30.1], [30.1, 30.1, 1.4],    # cell index 0 / 1
                     [2.1, 30.1, 30.1], [30.1, 63.3, 30.1], [30.1, 30.1, 63.6]], np.float32) * dx   # 2, 63 (4G - 1), 64 (4G)
    case = S._case(6, [S.model(S.FIXED_COROTATED, np.concatenate([inner, edge]), (0.0, 0.0, 0.0), dx)], [0])
    sim = S.build_engine(case)
    st = sim.stats()
    assert st.error & ERR_LOST, st.error
    kept = sim.particle_state(0)[:, :3]
    assert len(kept) == len(inner) + 3
    lost = edge[:4]
    assert np.min(np.abs(kept[:, None, :] - lost[None]).max(-1)) > 0
    sim.close()


def test_low_face_rule_kernel_level_entries_truncate(cuda_lib):
    """The drop-in entries keep the reference's truncating division: cell index 1 (cell - 2 = -1) lands in block 0, cell index
    0 (cell - 2 = -2) as well."""
    import torch
    import claymore_b200 as cb
    cfg = cb.Config(domain_bits=6)
    G = cfg.grid_size
    dx = cfg.dx
    pos = torch.tensor([[1.1 * dx, 30.1 * dx, 30.1 * dx], [0.2 * dx, 30.1 * dx, 30.1 * dx]], dtype=torch.float32, device="cuda")
    table = torch.full((G ** 3,), -1, dtype=torch.int32, device="cuda")
    keys = torch.zeros(3 * 64, dtype=torch.int32, device="cuda")
    count = torch.zeros(1, dtype=torch.int32, device="cuda")
    part = cb.Partition()
    part.count, part.index_table, part.active_keys = count.data_ptr(), table.data_ptr(), keys.data_ptr()
    assert cuda_lib.cb200_activate_blocks(C.byref(cfg), 2, pos.data_ptr(), part, None) == 0
    torch.cuda.synchronize()
    assert int(count.item()) == 1
    assert keys[:3].cpu().tolist() == [0, 7, 7]
    # the cell buckets put both particles into block 0, cells (3, 0, 0) and (2, 0, 0): (cell - 2) & 3 of -1 and -2
    mp = 128
    counts = torch.zeros(64, dtype=torch.int32, device="cuda")
    buckets = torch.zeros(64 * mp, dtype=torch.int32, device="cuda")
    pb = cb.ParticleBuffer()
    pb.material = cb.FIXED_COROTATED
    pb.cell_particle_counts, pb.cellbuckets = counts.data_ptr(), buckets.data_ptr()
    assert cuda_lib.cb200_build_particle_cell_buckets(C.byref(cfg), 2, pos.data_ptr(), pb, part, None) == 0
    torch.cuda.synchronize()
    c = counts.cpu().numpy()
    assert c.sum() == 2 and c[3 * 16] == 1 and c[2 * 16] == 1, np.nonzero(c)


def position_keys(p):
    """Exact integer keys of float32 positions on a 2^-20 lattice (the set-up positions are on it), for set comparisons."""
    return np.round(np.asarray(p, np.float64) * 2 ** 20).astype(np.int64) @ np.array([1 << 40, 1 << 20, 1], np.int64)


def test_cell_overflow_at_setup_is_flagged_and_clamped(cuda_lib):
    """A cell that receives more than max_ppc particles at set-up: kErrCellOverflow, the cell keeps max_ppc of them, the
    particle count is n - overflowed, and every other particle is unchanged."""
    dx = 1.0 / 64
    max_ppc = 8
    rest = S.box(dx, (20, 20, 20), (24, 24, 24))                                 # 8 per cell: full, not over
    crowd = (np.array([30.0, 30.0, 30.0]) + np.linspace(-0.3, 0.3, 13)[:, None]) * dx   # 13 particles in cell (30, 30, 30)
    case = S._case(6, [S.model(S.J_FLUID, np.concatenate([rest, crowd]).astype(np.float32), (0.0, 0.0, 0.0), dx)], [0], max_ppc=max_ppc)
    sim = S.build_engine(case)
    st = sim.stats()
    assert st.error == ERR_CELL_OVERFLOW, st.error
    s = sim.particle_state(0)
    assert len(s) == len(rest) + max_ppc
    in_rest = np.all(s[:, :3] < 25 * dx, axis=1)
    assert np.array_equal(np.sort(position_keys(s[in_rest, :3])), np.sort(position_keys(rest)))
    assert np.all(s[:, 3] == 1.0)
    sim.close()


def test_ninth_model_is_rejected(cuda_lib):
    from claymore_b200.simulator import GmpmSimulator
    from claymore_b200._capi import CB200Error
    dx = 1.0 / 64
    sim = GmpmSimulator(dt=1e-4, fps=0, config=S.config(S.CASES["fc_cube"]), max_blocks=1000)
    for i in range(8):
        sim.init_model(S.J_FLUID, S.box(dx, (20 + 3 * i, 20, 20), (22 + 3 * i, 22, 22)), (0.0, 0.0, 0.0))
    with pytest.raises(CB200Error):
        sim.init_model(S.J_FLUID, S.box(dx, (20, 30, 20), (22, 32, 22)), (0.0, 0.0, 0.0))
    sim.close()


# ---- kernel level: the drop-in entries on the oracle's containers ---------------------------------------------------------
def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _cb_buffer(cb, struct, tensors):
    pb = cb.ParticleBuffer()
    for f, _ in cb.ParticleBuffer._fields_:
        if f in tensors:
            setattr(pb, f, tensors[f].data_ptr())
        elif hasattr(struct, f):
            setattr(pb, f, getattr(struct, f))
    return pb


def _cb_partition(cb, tensors):
    p = cb.Partition()
    for f in ("count", "index_table", "active_keys"):
        setattr(p, f, tensors[f].data_ptr())
    return p


@pytest.mark.parametrize("material,deform", KERNEL_LEVEL)
def test_kernel_level_entries_match_ref64(oracle, cuda_lib, material, deform):
    """cb200_update_grid_velocity_query_max and the any-order cb200_g2p2g on copies of the oracle's containers, against ref64 with
    the oracle's kappa; with deform=True the particles carry F at det ~ 0.1, inverted, nearly singular and stretched, which
    sends FIXED_COROTATED's polar iteration to its SVD fall-back."""
    kernel_level_entries_check(oracle, cuda_lib, material, deform)


@pytest.mark.parametrize("case_step", KERNEL_LEVEL_CASES, ids=[f"{n}-{k}" + ("" if h else "-unhardened") for n, k, h in KERNEL_LEVEL_CASES])
def test_kernel_level_entries_match_ref64_cases(oracle, cuda_lib, case_step):
    """The same on scenes of the matrix: particles one ulp from cell faces (nodes with subnormal mass), a cell overflow inside the
    any-order g2p2g (the cell counts clamped at max_ppc, every particle's P2G kept), NACC with hardening_on = 0."""
    kernel_level_entries_check(oracle, cuda_lib, S.CASES[case_step[0]]["models"][0]["material"], False, case_step)


def kernel_level_entries_check(oracle, cuda_lib, material, deform, case_step=None):
    import torch
    import claymore_b200 as cb

    def cfg_of(osim):
        return cb.Config(domain_bits=osim.cfg.domain_bits, max_ppc=osim.cfg.max_ppc, gravity=osim.cfg.gravity)

    def grid_update(osim):
        _, nbc, _ = osim.block_counts()
        g = _dev(torch, osim.grid_array(0))
        keys = _dev(torch, osim.partition_arrays(0)["active_keys"])
        mv = torch.zeros(1, device="cuda")
        part = cb.Partition()
        part.active_keys = keys.data_ptr()
        assert cuda_lib.cb200_update_grid_velocity_query_max(C.byref(cfg_of(osim)), nbc, g.data_ptr(), part, osim.dt, mv.data_ptr(), None) == 0
        torch.cuda.synchronize()
        # the oracle's own update feeds g2p2g on both sides (S.kernel_level_inputs' contract)
        oracle.lib().orc_update_grid_velocity_query_max(C.byref(osim.cfg), nbc, oracle.ptr(osim.grid_array(0)), osim.partition_arrays(0)["struct"],
                                                        osim.dt, oracle.ptr(np.zeros(1, np.float32)))
        return g.cpu().numpy()[: nbc * 256], float(mv.item())

    def g2p2g(osim):
        pbc, nbc, ebc = osim.block_counts()
        cur, nxt = osim.buffer_arrays(0, 0), osim.buffer_arrays(0, 1)
        names = ("bins", "cell_particle_counts", "particle_bucket_sizes", "cellbuckets", "blockbuckets", "bin_offsets")
        t_cur = {k: _dev(torch, cur[k]) for k in names}
        t_nxt = {k: _dev(torch, nxt[k]) for k in names}
        t_nxt["cell_particle_counts"][: ebc * 64] = 0
        part = {k: _dev(torch, v) for k, v in osim.partition_arrays(0).items() if k != "struct"}
        prev = {k: _dev(torch, v) for k, v in osim.partition_arrays(1).items() if k != "struct"}
        g0 = _dev(torch, osim.grid_array(0))
        g1 = torch.zeros_like(g0)
        assert cuda_lib.cb200_g2p2g(C.byref(cfg_of(osim)), osim.dt, osim.dt, pbc, _cb_buffer(cb, cur["struct"], t_cur), _cb_buffer(cb, nxt["struct"], t_nxt),
                                    _cb_partition(cb, prev), _cb_partition(cb, part), g0.data_ptr(), g1.data_ptr(), None) == 0
        torch.cuda.synchronize()
        return g1.cpu().numpy()[: nbc * 256], t_nxt["bins"].cpu().numpy(), t_nxt["cell_particle_counts"].cpu().numpy()[: ebc * 64]

    kernel_level_check(oracle, material, deform, grid_update, g2p2g, f"cb200 kernel level {material} {deform} {case_step}", case_step)


def test_kernel_level_rasterize_matches_ref64(oracle, cuda_lib):
    """cb200_rasterize (per-particle atomics) of every model of multi_model_8 and high_faces into the oracle's set-up partition,
    against ref64.rasterize with the kappa of set-up rasterisation."""
    import torch
    import claymore_b200 as cb
    for name in ("multi_model_8", "high_faces"):
        case = S.CASES[name]
        osim = S.build_oracle(oracle, case)
        _, nbc, _ = osim.block_counts()
        p = osim.partition_arrays(0)
        t = {k: _dev(torch, v) for k, v in p.items() if k != "struct"}
        g = torch.zeros(nbc * 256, device="cuda")
        cfg = cb.Config(domain_bits=case["domain_bits"], max_ppc=case["max_ppc"])
        for m in case["models"]:
            pos = _dev(torch, m["pos"])
            v0 = np.array(m["v0"], np.float32)
            assert cuda_lib.cb200_rasterize(C.byref(cfg), len(m["pos"]), pos.data_ptr(), g.data_ptr(), _cb_partition(cb, t), S.ref_params(m)["mass"],
                                            v0.ctypes.data_as(C.c_void_p), None) == 0
        torch.cuda.synchronize()
        keys, grid, mag = ref64.rasterize(osim.cfg, [dict(pos=m["pos"], v0=m["v0"], mass=S.ref_params(m)["mass"]) for m in case["models"]])
        r = dict(keys=keys, grid=grid, mag=mag, stress=np.zeros_like(grid), models=[])
        rep = ref64.compare(r, p["active_keys"].reshape(-1, 3)[:nbc], g.cpu().numpy().reshape(nbc, 4, 64), [], RASTER_KAPPA, 0.0, [])
        check_report(rep, f"{name} cb200_rasterize")
        osim.close()
