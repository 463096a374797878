"""GPU tests of the particle read-outs' row order.

retrieve, particle_state and the checkpoint (and through it the emission) gather rows with one device routine, in one order:
particle blocks in partition order, then bucket order inside a block.  So, with no sorting, particle_state(m) is byte for byte
model m's section of a checkpoint of the same state, every form of retrieve(m) is its first three columns bit for bit, and two
read-outs of an unchanged simulator return the same bytes: after a set-up, after sub-steps that move particles across cell faces
(advection tags other than the identity), with two models in shared blocks, after an emission and after a restore.
"""
import numpy as np
import pytest
import torch

import scenes
from claymore_b200 import checkpoint, samplers
from test_gpu_checkpoint import _restored

pytestmark = pytest.mark.gpu

DX = 1.0 / 64


def _check_read_outs(sim, label):
    blob = sim.save_checkpoint()
    states = checkpoint.read(blob)["states"]
    assert len(states) == len(sim.counts), label
    for m in range(len(sim.counts)):
        st = sim.particle_state(m)
        assert len(st) > 0, label
        assert st.tobytes() == states[m].tobytes(), f"{label}: particle_state({m}) vs checkpoint"
        assert sim.particle_state(m).tobytes() == st.tobytes(), f"{label}: particle_state({m}) twice"
        pos = np.ascontiguousarray(st[:, :3]).tobytes()
        assert sim.retrieve(m).tobytes() == pos, f"{label}: retrieve({m})"
        assert sim.retrieve(m, copy=False).tobytes() == pos, f"{label}: retrieve({m}, copy=False)"
        pinned = torch.empty((sim.counts[m], 3), dtype=torch.float32).pin_memory().numpy()
        assert sim.retrieve(m, out=pinned).tobytes() == pos, f"{label}: retrieve({m}, out=pinned)"
    assert sim.save_checkpoint().tobytes() == blob.tobytes(), f"{label}: checkpoint twice"


def _cells(sim, m):
    return np.sort(scenes.key_hash(np.floor(sim.particle_state(m)[:, :3] / DX).astype(np.int64)))


def _substeps_cross_cells(sim, k):
    before = [_cells(sim, m) for m in range(len(sim.counts))]
    sim.step(k)
    assert sim.stats().error == 0
    assert any(not np.array_equal(b, _cells(sim, m)) for m, b in enumerate(before)), "no particle changed its cell"


@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
@pytest.mark.parametrize("material", [scenes.FIXED_COROTATED, scenes.J_FLUID, scenes.SAND, scenes.NACC])
def test_read_outs_share_one_order(cuda_lib, material, use_graph):
    # 48^3 cells (1728 particle blocks) moving half a cell in ten sub-steps
    sim = scenes.build_engine(scenes.small_cube(lo=8, hi=56, material=material, v0=(2.0, -8.0, 1.0)), max_blocks=6000, use_graph=use_graph)
    _check_read_outs(sim, "set-up")
    _substeps_cross_cells(sim, 10)
    _check_read_outs(sim, "10 sub-steps")
    sim.close()


@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
def test_shared_blocks_emission_and_restore(cuda_lib, use_graph):
    # the boxes meet inside the particle blocks of cells x = 28..31
    models = [dict(material=scenes.J_FLUID, pos=samplers.uniform_box(DX, (8, 8, 8), (30, 40, 40)), v0=(2.0, -8.0, 1.0)),
              dict(material=scenes.SAND, pos=samplers.uniform_box(DX, (30, 8, 8), (52, 40, 40)), v0=(-2.0, -8.0, 1.0))]
    sim = scenes.build_engine(dict(domain_bits=6, models=models), max_blocks=6000, use_graph=use_graph)
    _check_read_outs(sim, "set-up")
    _substeps_cross_cells(sim, 10)
    _check_read_outs(sim, "10 sub-steps")
    add = samplers.uniform_box(DX, (24, 44, 20), (36, 52, 28))
    assert sim.add_particles(1, add, (0.0, -8.0, 0.0)) == len(add)
    _check_read_outs(sim, "after add_particles")
    _substeps_cross_cells(sim, 5)
    _check_read_outs(sim, "5 sub-steps after add_particles")
    r = _restored(sim.save_checkpoint(), use_graph=use_graph)
    _check_read_outs(r, "restored")
    _substeps_cross_cells(r, 5)
    _check_read_outs(r, "5 sub-steps after the restore")
    r.close()
    sim.close()
