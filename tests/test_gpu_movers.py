"""GPU parity for particles that change cell in a sub-step ("movers"), against the CPU oracle.

The lattice scenes place particles at +-0.25 dx (27 per cell: -1/3, 0, +1/3 dx) around the cell centre and translate them
rigidly, so a whole sub-lattice crosses a cell face in the same sub-step, the one the velocity is chosen for.  g2p2g accumulates
a mover whose new cell lies in its particle block with that cell's particles, and scatters the rest (movers leaving the block,
and in the step driver's fixed-corotated path arrivals beyond a cell's list) with shared-memory atomics: both kinds occur in every
scene here.
Tolerances are those of test_gpu_parity.py.
"""
import ctypes as C

import numpy as np
import pytest

import scenes
from test_gpu_parity import _cb_buffer, _compare_state, _dev, _torch

pytestmark = pytest.mark.gpu

MATERIALS = [scenes.FIXED_COROTATED, scenes.J_FLUID, scenes.SAND, scenes.NACC]
DT = 1e-4
DIRECTIONS = {"+x": (1.0, 0.0, 0.0), "-y": (0.0, -1.0, 0.0), "xyz": (1.0, 1.0, 1.0)}


def _crossing_velocity(direction, gap, substep, domain_bits=6):
    """Velocity that carries a particle `gap` cells short of a face across it in sub-step `substep` (mid-way through it)."""
    dx = 1.0 / (1 << domain_bits)
    speed = gap * dx / ((substep - 0.5) * DT)
    return tuple(speed * c for c in direction)


def _step_and_compare(oracle, scene, substep, **tol):
    """Both simulators up to the sub-step before the crossing, then compared after it, the crossing one and the next."""
    osim = scenes.build_oracle(oracle, scene, dt=DT)
    esim = scenes.build_engine(scene, dt=DT)
    osim.step(substep - 2)
    esim.step(substep - 2)
    for k in (substep - 1, substep, substep + 1):
        osim.step(1)
        esim.step(1)
        _compare_state(osim, esim, 1, f"after sub-step {k} (crossing in {substep})", **tol)
    esim.close()


@pytest.mark.parametrize("material", MATERIALS)
@pytest.mark.parametrize("direction", list(DIRECTIONS))
@pytest.mark.parametrize("cells", [(20, 32), (21, 31)])
def test_sublattice_crossing_matches_oracle(oracle, cuda_lib, material, direction, cells):
    # the +0.25 dx sub-lattice is 0.25 cells from the face ahead of it; the cube spans several particle blocks.  With faces on
    # block boundaries (20..32) the movers crossing the cube's faces leave their block; with faces inside blocks (21..31) they
    # arrive in empty cells of their own block, whose phase-2 threads have no home particles
    v0 = _crossing_velocity(DIRECTIONS[direction], 0.25, 4)
    _step_and_compare(oracle, scenes.small_cube(lo=cells[0], hi=cells[1], material=material, v0=v0), 4)


@pytest.mark.parametrize("material", MATERIALS)
def test_dense_crossing_overflows_arrival_lists(oracle, cuda_lib, material):
    # 27 per cell: the +1/3 dx sub-lattice (9 particles of every cell) is 1/6 cell from the face ahead, so 9 movers land in each cell
    v0 = _crossing_velocity((1.0, 0.0, 0.0), 1.0 / 6.0, 3)
    _step_and_compare(oracle, scenes.dense_cube(material=material, v0=v0), 3, pos_tol=5e-6, f_tol=2e-4)


@pytest.mark.parametrize("material", MATERIALS)
@pytest.mark.parametrize("direction", list(DIRECTIONS))
def test_g2p2g_kernel_sublattice_crossing(oracle, cuda_lib, material, direction):
    """cb200_g2p2g (any bucket order, counting-sorted in the kernel) against orc_g2p2g on the sub-step of a crossing: same
    containers in, same containers out, compared as test_g2p2g_kernel_differential compares them."""
    torch = _torch()
    import claymore_b200 as cb
    ob = oracle
    steps_before = 4
    scene = scenes.small_cube(material=material, v0=_crossing_velocity(DIRECTIONS[direction], 0.25, steps_before + 1))
    osim = scenes.build_oracle(ob, scene, dt=DT)
    osim.step(steps_before)
    pbc, nbc, ebc = osim.block_counts()
    cfg_o = osim.cfg
    cfg_c = cb.Config(domain_bits=cfg_o.domain_bits, max_ppc=cfg_o.max_ppc)
    dt = osim.dt
    cur, nxt = osim.buffer_arrays(0, 0), osim.buffer_arrays(0, 1)
    part, prev = osim.partition_arrays(0), osim.partition_arrays(1)
    g0, g1 = osim.grid_array(0), osim.grid_array(1)
    mv = np.zeros(1, np.float32)
    ob.lib().orc_update_grid_velocity_query_max(C.byref(cfg_o), nbc, ob.ptr(g0), part["struct"], dt, ob.ptr(mv))
    g1[: nbc * 256] = 0
    nxt["cell_particle_counts"][: ebc * 64] = 0
    keys = ("bins", "cell_particle_counts", "particle_bucket_sizes", "cellbuckets", "blockbuckets", "bin_offsets")
    t_cur = {k: _dev(torch, cur[k]) for k in keys}
    t_nxt = {k: _dev(torch, nxt[k]) for k in keys}
    t_part = {k: _dev(torch, part[k]) for k in ("count", "index_table", "active_keys")}
    t_prev = {k: _dev(torch, prev[k]) for k in ("count", "index_table", "active_keys")}
    t_g0, t_g1 = _dev(torch, g0), _dev(torch, g1)
    c_cur, c_nxt = _cb_buffer(cb, cur["struct"], t_cur), _cb_buffer(cb, nxt["struct"], t_nxt)
    c_part, c_prev = cb.Partition(), cb.Partition()
    for name in ("count", "index_table", "active_keys"):
        setattr(c_part, name, t_part[name].data_ptr())
        setattr(c_prev, name, t_prev[name].data_ptr())
    err = cuda_lib.cb200_g2p2g(C.byref(cfg_c), dt, dt, pbc, c_cur, c_nxt, c_prev, c_part, t_g0.data_ptr(), t_g1.data_ptr(), None)
    assert err == 0
    torch.cuda.synchronize()
    ob.lib().orc_g2p2g(C.byref(cfg_o), dt, dt, pbc, cur["struct"], nxt["struct"], prev["struct"], part["struct"], ob.ptr(g0), ob.ptr(g1))
    # a sub-lattice changed cell in this sub-step: an eighth of the particles are re-bucketed away from their old cell
    cc_c, cc_o = t_nxt["cell_particle_counts"].cpu().numpy()[: ebc * 64], nxt["cell_particle_counts"][: ebc * 64]
    assert np.array_equal(cc_c, cc_o)
    assert np.count_nonzero(cc_o % 8) > 0, "no particle changed cell: the scene misses its crossing"
    # next bins slot for slot, cell buckets as sets per cell
    bins_c, bins_o = t_nxt["bins"].cpu().numpy(), nxt["bins"]
    bf, nch = ob.BIN_FLOATS[material], ob.CHANNELS[material]
    offs, sizes = nxt["bin_offsets"], nxt["particle_bucket_sizes"]
    worst_pos = worst_f = 0.0
    for b in range(pbc):
        n = int(sizes[b])
        for bi in range((n + 31) // 32):
            lanes = min(32, n - 32 * bi)
            o = (int(offs[b]) + bi) * bf
            x = bins_c[o:o + nch * 32].reshape(nch, 32)[:, :lanes]
            r = bins_o[o:o + nch * 32].reshape(nch, 32)[:, :lanes]
            worst_pos = max(worst_pos, np.abs(x[:3] - r[:3]).max())
            if nch > 3:
                worst_f = max(worst_f, np.abs(x[3:] - r[3:]).max())
    assert worst_pos <= 1e-6, worst_pos
    assert worst_f <= 2e-5, worst_f
    cb_c, cb_o = t_nxt["cellbuckets"].cpu().numpy(), nxt["cellbuckets"]
    mp = cfg_o.max_ppc
    for cell in np.nonzero(cc_o)[0]:
        n = cc_o[cell]
        assert np.array_equal(np.sort(cb_c[cell * mp: cell * mp + n]), np.sort(cb_o[cell * mp: cell * mp + n]))
    # next grid per cell
    gc, go = t_g1.cpu().numpy()[: nbc * 256].reshape(nbc, 4, 64), g1[: nbc * 256].reshape(nbc, 4, 64)
    assert np.allclose(gc[:, 0], go[:, 0], rtol=1e-5, atol=1e-5 * go[:, 0].max())
    assert np.abs(gc[:, 1:] - go[:, 1:]).max() <= 1e-4 * np.abs(go[:, 1:]).max()
