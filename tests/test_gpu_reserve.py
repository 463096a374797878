"""GPU tests of growing the block capacity in place (cb200_sim_reserve, GmpmSimulator.reserve).

Growth keeps every live array's contents: a reserve between sub-steps changes nothing that describes the state, bit for bit, and a
grown simulator takes particles exactly as one that was not grown, which reads the kept cell offsets and bucket sizes.
"""
import numpy as np
import pytest

from claymore_b200 import checkpoint
from test_gpu_checkpoint import _restored, _sorted_rows
from test_gpu_emit import _cell_centres, _mid_run_case
import ref64_cases as S

pytestmark = pytest.mark.gpu


def _live(sim):
    """the checkpoint (its header as a dict, the raw data sections), every model's particle state (sorted: the gather's order is not
    fixed), the active keys and grid[0]"""
    blob = sim.save_checkpoint()
    head = checkpoint.info(blob)
    data = blob[head["models"][0]["offset"]:].tobytes()
    states = [_sorted_rows(sim.particle_state(m)).tobytes() for m in range(len(sim.materials))]
    return head, data, states, sim.active_keys().tobytes(), sim.grid().tobytes()


@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
def test_reserve_keeps_the_live_state(cuda_lib, use_graph):
    sim = S.build_engine(_mid_run_case(), use_graph=use_graph)
    sim.step(10)
    cap = sim.capacity()[0]
    head, data, states, keys, grid = _live(sim)
    sim.reserve(2 * cap)
    assert sim.capacity()[0] == 2 * cap
    head2, data2, states2, keys2, grid2 = _live(sim)
    assert (head["max_blocks"], head2["max_blocks"]) == (cap, 2 * cap)
    head2["max_blocks"] = cap
    assert head2 == head
    assert data2 == data, "checkpoint data sections"
    for m, (a, b) in enumerate(zip(states, states2)):
        assert a == b, f"model {m} particle state"
    assert keys2 == keys, "active keys"
    assert grid2 == grid, "grid"
    sim.step(5)
    assert sim.stats().error == 0
    sim.close()


def test_reserve_then_emission_adds_what_the_unreserved_adds(cuda_lib):
    sim = S.build_engine(_mid_run_case())
    sim.step(10)
    blob = sim.save_checkpoint()
    sim.close()
    kept, grown = _restored(blob), _restored(blob)
    grown.reserve(2 * grown.capacity()[0])
    cand = _cell_centres((10, 16, 16), (50, 46, 40))
    added = [s.add_particles(1, cand, (0.0, -1.0, 0.0), fill="empty") for s in (kept, grown)]
    assert 0 < added[0] < len(cand)
    assert added[1] == added[0]
    assert grown.block_counts() == kept.block_counts()
    for m in range(len(kept.materials)):
        assert _sorted_rows(grown.particle_state(m)).tobytes() == _sorted_rows(kept.particle_state(m)).tobytes(), f"model {m}"
    grown.step(5)
    assert grown.stats().error == 0
    kept.close()
    grown.close()
