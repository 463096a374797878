"""GPU tests of the step driver's cell-bucket layout at the driver level.

The driver keeps its cell buckets slot-grouped (grouped_cell_slot in common.cuh): set-up, restore and emission write them with
build_particle_cell_buckets_kernel<true>, g2p2g's re-bucketing stores its tags there, and the rebuild and set-up flatten read them.
If a writer and the flatten disagree on the layout, a block bucket picks up stale or foreign tags.  What the sorted g2p2g relies
on is checked through a checkpoint, whose rows come out in partition order and then bucket order (DESIGN section 2.5):

* split into runs by the bucket block of their position (floor semantics, as the driver), every block is one run;
* inside a run the bucketing cell never decreases (cell-major buckets);
* every run holds, per cell, as many rows as there are positions in that cell;
* every particle is there exactly once (no duplicate rows, no row of a lost particle).

Scenes: lattices with 1 to max_ppc particles per cell (tags in every slot group, at 128 in the last one), a dense scene at 27 per
cell, and a moving lattice of 8 to 27 per cell that re-buckets particles across block faces and into slots beyond eight.
"""
import numpy as np
import pytest

import scenes
from claymore_b200 import checkpoint
from claymore_b200.simulator import GmpmSimulator

pytestmark = pytest.mark.gpu

DOMAIN_BITS = 6
DX = 1.0 / (1 << DOMAIN_BITS)


def _cell_lattice(max_ppc, lo=20, cells=(8, 8, 6)):
    """cells (lo + i, lo + j, lo + k), the c-th of them holding 1 + c % max_ppc particles on a small lattice around its centre"""
    pos = []
    c = 0
    for i in range(cells[0]):
        for j in range(cells[1]):
            for k in range(cells[2]):
                n = 1 + c % max_ppc
                c += 1
                side = int(np.ceil(n ** (1.0 / 3.0) - 1e-9))
                sub = (np.arange(side) - (side - 1) / 2) * (0.7 / side)
                off = np.stack(np.meshgrid(sub, sub, sub, indexing="ij"), axis=-1).reshape(-1, 3)[:n]
                pos.append((np.array([lo + i, lo + j, lo + k], np.float64) + off) * DX)
    return np.concatenate(pos).astype(np.float32)


def _crossing_lattice(lo=18.0, hi=30.0, spacing=0.4):
    """a lattice 0.4 dx apart (8 to 27 particles per cell) that moves about 0.2 dx per sub-step: across cell and block faces"""
    ax = np.arange(lo, hi, spacing) * DX
    return np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), axis=-1).reshape(-1, 3).astype(np.float32)


SCENES = {
    "ppc1to8": (lambda: _cell_lattice(8), (0.0, 0.0, 0.0), 8),
    "ppc1to16": (lambda: _cell_lattice(16), (0.0, 0.0, 0.0), 16),
    "ppc1to128": (lambda: _cell_lattice(128), (0.0, 0.0, 0.0), 128),
    "dense27": (lambda: scenes.dense_cube()["models"][0]["pos"], (0.4, -0.8, 0.3), 32),
    "crossing": (_crossing_lattice, (16.0, -24.0, 12.0), 32),
}


def _bucket_of(pos):
    """(block key hash, cell in block) of each position, as the driver buckets it: cell index round-half-away(p / dx) - 2, block by floor"""
    c = np.floor(pos.astype(np.float64) * (1 << DOMAIN_BITS) + 0.5).astype(np.int64) - 2
    blk = c >> 2
    key = (blk[:, 0] << 40) + (blk[:, 1] << 20) + blk[:, 2]
    cell = (c[:, 0] & 3) * 16 + (c[:, 1] & 3) * 4 + (c[:, 2] & 3)
    return key, cell


def _check_layout(sim, label):
    st = sim.stats()
    assert st.error == 0, f"{label}: engine error bits {st.error}"
    for m, rows in enumerate(checkpoint.read(sim.save_checkpoint())["states"]):
        tag = f"{label}, model {m}"
        pos = rows[:, :3]
        assert len(rows) == sim.counts[m], f"{tag}: {len(rows)} rows for {sim.counts[m]} particles"
        assert (np.abs(pos).sum(1) > 0).all(), f"{tag}: a row of a lost particle"
        assert len(np.unique(rows, axis=0)) == len(rows), f"{tag}: a particle appears more than once"
        key, cell = _bucket_of(pos)
        starts = np.flatnonzero(np.r_[True, key[1:] != key[:-1]])
        assert len(np.unique(key[starts])) == len(starts), f"{tag}: a block's rows are not one run"
        ends = np.r_[starts[1:], len(key)]
        # cell-major inside every run: the cell never decreases except where a new run starts
        step = np.diff(cell)
        inside = np.ones(len(step), bool)
        inside[starts[1:] - 1] = False
        assert (step[inside] >= 0).all(), f"{tag}: a bucket is not cell-major"
        # per-cell counts of each run against a count of all positions
        want = {}
        for k, c in zip(key, cell):
            want[(int(k), int(c))] = want.get((int(k), int(c)), 0) + 1
        for s, e in zip(starts, ends):
            cells, counts = np.unique(cell[s:e], return_counts=True)
            for c, n in zip(cells, counts):
                assert n == want[(int(key[s]), int(c))], f"{tag}: cell {int(c)} of a block holds {n} rows"


@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
@pytest.mark.parametrize("name", list(SCENES))
def test_bucket_order_after_sub_steps(cuda_lib, name, use_graph):
    make, v0, max_ppc = SCENES[name]
    scene = dict(domain_bits=DOMAIN_BITS, models=[dict(material=scenes.FIXED_COROTATED, pos=make(), v0=v0)])
    sim = scenes.build_engine(scene, max_ppc=max_ppc, use_graph=use_graph)
    try:
        _check_layout(sim, f"{name}: set-up")
        for s in range(1, 9):
            sim.step(1)
            if s in (1, 2, 4, 8):
                _check_layout(sim, f"{name}: sub-step {s}")
    finally:
        sim.close()


@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
@pytest.mark.parametrize("name", ["ppc1to16", "crossing"])
def test_bucket_order_after_emission_and_restore(cuda_lib, name, use_graph):
    make, v0, max_ppc = SCENES[name]
    pos = make()
    scene = dict(domain_bits=DOMAIN_BITS, models=[dict(material=scenes.FIXED_COROTATED, pos=pos, v0=v0)])
    sim = scenes.build_engine(scene, max_ppc=max_ppc, use_graph=use_graph)
    try:
        sim.step(3)
        # a second copy of the scene, shifted by four blocks: new blocks and cells, bucketed through the set-up path
        assert sim.add_particles(0, pos + np.float32(16 * DX), v0=v0) == len(pos)
        _check_layout(sim, f"{name}: emission")
        sim.step(2)
        _check_layout(sim, f"{name}: emission + 2 sub-steps")
        blob = sim.save_checkpoint()
    finally:
        sim.close()
    r = GmpmSimulator.from_checkpoint(blob, use_graph=use_graph)
    try:
        r.restore(blob)
        _check_layout(r, f"{name}: restore")
        r.step(2)
        _check_layout(r, f"{name}: restore + 2 sub-steps")
    finally:
        r.close()
