"""GPU tests of checkpoint / restore: the snapshot and restore kernels and the step driver's checkpoint_begin / _end / restore.

A round trip (checkpoint, restore into a fresh simulator) is exact: block counts, key sets per class, the clock, the grid by key
and the particle states as sorted rows are bitwise equal, and a checkpoint of the restored simulator equals the original once
canonically ordered.  A continuation (k sub-steps, checkpoint, destroy, restore, m sub-steps) differs from an uninterrupted run
only by the order of floating-point sums in P2G, so it is held to the bounds of the parity tests (test_gpu_parity._compare_state,
test_gpu_collider, test_gpu_scale) against the CPU oracle and against the uninterrupted engine.
"""
import threading

import numpy as np
import pytest

import collider_oracle_binding as cob
import scenes
from claymore_b200 import checkpoint, mgsp
from claymore_b200._capi import CB200Error, Config
from claymore_b200.simulator import GmpmSimulator
from test_gpu_collider import _compare_state as _compare_collider, _fields, _params, _set_both
from test_gpu_parity import _compare_state
from test_gpu_scale import _compare_with_live_oracle

pytestmark = pytest.mark.gpu


def _sorted_rows(a):
    return a[np.lexsort(a.T[::-1])]


def _canonical(blob):
    d = checkpoint.read(blob)
    o = np.argsort(scenes.key_hash(d["keys"]))
    head = {k: v for k, v in d.items() if k not in ("states", "keys", "grid")}
    return head, [_sorted_rows(s) for s in d["states"]], d["keys"][o], d["grid"][o]


def _restored(blob, **kw):
    sim = GmpmSimulator.from_checkpoint(blob, **kw)
    sim.restore(blob)
    return sim


def _assert_round_trip(a, b, nmodels):
    sa, sb = a.stats(), b.stats()
    assert sa.error == 0 and sb.error == 0
    counts = (sa.particle_block_count, sa.neighbor_block_count, sa.exterior_block_count)
    assert counts == (sb.particle_block_count, sb.neighbor_block_count, sb.exterior_block_count)
    ka, kb = a.active_keys(), b.active_keys()
    pbc, nbc, ebc = counts
    for lo, hi in ((0, pbc), (pbc, nbc), (nbc, ebc)):
        assert np.array_equal(np.sort(scenes.key_hash(ka[lo:hi])), np.sort(scenes.key_hash(kb[lo:hi]))), (lo, hi)
    for f in ("dt", "next_dt", "step_time", "steps"):
        assert getattr(sa, f) == getattr(sb, f), f
    assert a.sim_time() == b.sim_time()
    ha, ga = scenes.grid_by_key(ka, a.grid())
    hb, gb = scenes.grid_by_key(kb, b.grid())
    assert np.array_equal(ha, hb) and ga.tobytes() == gb.tobytes()
    for m in range(nmodels):
        assert _sorted_rows(a.particle_state(m)).tobytes() == _sorted_rows(b.particle_state(m)).tobytes()


def _canonical_equal(x, y):
    hx, sx, kx, gx = _canonical(x)
    hy, sy, ky, gy = _canonical(y)
    assert hx == hy
    assert all(a.tobytes() == b.tobytes() for a, b in zip(sx, sy))
    assert kx.tobytes() == ky.tobytes() and gx.tobytes() == gy.tobytes()


@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
@pytest.mark.parametrize("material", [scenes.FIXED_COROTATED, scenes.J_FLUID, scenes.SAND, scenes.NACC])
def test_round_trip_is_exact(cuda_lib, material, use_graph):
    esim = scenes.build_engine(scenes.small_cube(material=material), use_graph=use_graph)
    esim.step(7)
    blob = esim.save_checkpoint()
    inf = checkpoint.info(blob)
    assert inf["steps"] == 7 and inf["models"][0]["count"] == 13824 and inf["bytes"] == len(blob)
    r = _restored(blob, use_graph=use_graph)
    _assert_round_trip(esim, r, 1)
    _canonical_equal(blob, r.save_checkpoint())
    r.close()
    esim.close()


def test_snapshots_are_deterministic_and_overlap_substeps(cuda_lib):
    esim = scenes.build_engine(scenes.two_cubes_colliding(), dt=2e-4)
    esim.step(7)
    a = esim.save_checkpoint()
    b = esim.save_checkpoint()
    assert a.tobytes() == b.tobytes()
    esim.checkpoint_begin()
    esim.step(5)           # runs while the copy of the snapshot is in flight
    c = esim.checkpoint_end()
    assert c.tobytes() == a.tobytes()
    assert esim.stats().steps == 12
    esim.close()


def _mixed_scene(domain_bits=6):
    """fluid + sand + fixed-corotated cubes side by side: three g2p2g launches per sub-step"""
    dx = 1.0 / (1 << domain_bits)
    from claymore_b200 import samplers
    boxes = [(scenes.J_FLUID, (14, 20, 20), (0.5, -0.5, 0.0)), (scenes.SAND, (26, 22, 20), (0.0, -0.8, 0.2)), (scenes.FIXED_COROTATED, (38, 20, 22), (-0.5, -0.3, 0.0))]
    return dict(domain_bits=domain_bits, models=[dict(material=m, pos=samplers.uniform_box(dx, lo, tuple(c + 8 for c in lo)), v0=v) for m, lo, v in boxes])


CONTINUATIONS = {
    "fc": (lambda: scenes.small_cube(material=scenes.FIXED_COROTATED), 1e-4, 7, 8, {}),
    "fluid": (lambda: scenes.small_cube(material=scenes.J_FLUID), 1e-4, 7, 8, {}),
    "sand": (lambda: scenes.small_cube(material=scenes.SAND), 1e-4, 7, 8, {}),
    "nacc": (lambda: scenes.small_cube(material=scenes.NACC), 1e-4, 7, 8, {}),
    "two_colliding": (scenes.two_cubes_colliding, 2e-4, 20, 20, dict(pos_tol=5e-6, f_tol=2e-4)),
    "fluid_sand_fc": (_mixed_scene, 1e-4, 10, 10, dict(pos_tol=5e-6, f_tol=2e-4)),
}


@pytest.mark.parametrize("name", sorted(CONTINUATIONS))
def test_continuation_matches_oracle_and_uninterrupted_engine(oracle, cuda_lib, name):
    make, dt, k, m, tol = CONTINUATIONS[name]
    scene = make()
    n = len(scene["models"])
    osim = scenes.build_oracle(oracle, scene, dt=dt)
    whole = scenes.build_engine(scene, dt=dt)
    esim = scenes.build_engine(scene, dt=dt)
    esim.step(k)
    blob = esim.save_checkpoint()
    esim.close()
    r = _restored(blob)
    osim.step(k + m)
    whole.step(k + m)
    r.step(m)
    _compare_state(osim, r, n, f"{name}: {k} + {m} sub-steps vs oracle", **tol)
    _compare_state(whole, r, n, f"{name}: {k} + {m} sub-steps vs uninterrupted engine", **tol)
    assert r.stats().steps == k + m and r.sim_time() == whole.sim_time()
    r.close()
    whole.close()


def test_frames_resume_where_they_stopped(cuda_lib):
    scene = scenes.small_cube()
    fps, dt = 240, 1e-4
    whole = scenes.build_engine(scene, dt=dt, fps=fps)
    whole.nframes = 4
    whole.advance_frame()
    whole.advance_frame()
    after2 = whole.save_checkpoint()
    assert checkpoint.info(after2)["frames"] == 2
    whole.advance_frame()
    r = _restored(after2)
    assert r.cur_frame == 2
    r.advance_frame()
    assert checkpoint.info(r.save_checkpoint())["frames"] == 3
    for f in ("steps", "step_time", "dt"):
        assert getattr(r.stats(), f) == getattr(whole.stats(), f), f
    assert r.sim_time() == whole.sim_time()
    _compare_state(whole, r, 1, "frame 3 after a resume at frame 2", pos_tol=5e-6, f_tol=2e-4)
    # main_loop on a restored simulator runs only the remaining frames
    whole.advance_frame()
    m = _restored(after2, frames=4)
    seen = []
    m.main_loop(on_frame=lambda sim, f: seen.append(f))
    assert seen == [3, 4]
    assert m.sim_time() == whole.sim_time() and m.stats().steps == whole.stats().steps
    # mid-frame: the device frame clock (step with fps > 0) continues where it was
    a = scenes.build_engine(scene, dt=dt, fps=fps)
    a.step(50)                      # 42 sub-steps per frame: inside the second frame
    mid = a.save_checkpoint()
    a.step(40)
    b = _restored(mid)
    b.step(40)
    for f in ("steps", "step_time", "dt", "next_dt"):
        assert getattr(b.stats(), f) == getattr(a.stats(), f), f
    assert b.sim_time() == a.sim_time()
    _compare_state(a, b, 1, "mid-frame resume", pos_tol=5e-6, f_tol=2e-4)
    for s in (whole, r, m, a, b):
        s.close()


@pytest.mark.timeout(600)
def test_moving_paddle_resumes_where_it_was(oracle, cuda_lib):
    scene = scenes.small_cube(material=scenes.J_FLUID, lo=18, hi=34, v0=(0.0, 0.0, 0.0))
    osim = scenes.build_oracle(oracle, scene, sim_class=cob.ColliderOracleSim)
    esim = scenes.build_engine(scene)
    p = dict(_params("slip", 0.0, "static"), trans=(-0.08, 0.0, 0.0), trans_vel=(1.5, 0.0, 0.0))
    sdf, grad = _set_both(osim, esim, scene["domain_bits"], "box", p)
    esim.step(20)
    blob = esim.save_checkpoint()
    esim.close()
    r = GmpmSimulator.from_checkpoint(blob)
    r.set_collider(sdf, grad, **p)     # the field is a scene input: set before the restore
    r.restore(blob)
    osim.step(20)
    _compare_collider(osim, r, "paddle at the checkpoint")
    for k in range(2):
        osim.step(10)
        r.step(10)
        _compare_collider(osim, r, f"paddle {10 * (k + 1)} sub-steps after the resume")
    assert r.sim_time() == pytest.approx(osim.sim_time, rel=1e-6)
    r.close()


def _threads(fn, sims):
    errs = []

    def run(s):
        try:
            fn(s)
        except Exception as e:  # pragma: no cover
            errs.append(e)
    th = [threading.Thread(target=run, args=(s,)) for s in sims]
    [t.start() for t in th]
    [t.join(120) for t in th]
    assert not errs and not any(t.is_alive() for t in th), errs


def _check_mgsp(osim, sims, label, dt_default):
    """test_gpu_parity.test_mgsp_two_shards_match_single_domain's check(): the shards' grids sum to the single domain's, halo blocks
    hold the full sum on both owners, and the union of the shards' particles is the single domain's."""
    okeys, ogrid = osim.active_keys(), osim.grid()
    oh, og = scenes.grid_by_key(okeys, ogrid)
    lut = {int(h): i for i, h in enumerate(oh)}
    total = np.zeros_like(og)
    seen = np.zeros(len(og), bool)
    sets = []
    for s in sims:
        assert s.stats().error == 0, label
        k, g = s.active_keys(), s.grid()
        sets.append(set(int(h) for h in scenes.key_hash(k[: len(g)])))
    common = sets[0] & sets[1]
    assert len(common) > 0
    scale = np.abs(og).max(axis=(0, 2), keepdims=True)
    for s in sims:
        k, g = s.active_keys(), s.grid()
        for b, h in enumerate(scenes.key_hash(k[: len(g)])):
            i = lut.get(int(h))
            if i is None:
                assert np.abs(g[b]).max() == 0, label
                continue
            if int(h) in common:
                assert np.all(np.abs(g[b] - og[i]) <= 2e-4 * scale[0] + 1e-12), (label, "halo block")
                if not seen[i]:
                    total[i] = g[b]
            else:
                total[i] += g[b]
            seen[i] = True
    assert np.all(np.abs(total - og) <= 2e-4 * scale + 1e-12), label
    so = osim.particle_state(0)
    se = np.concatenate([s.particle_state(0) for s in sims])
    assert len(so) == len(se)
    loose = dt_default > 5e-4
    idx = scenes.match_particles(so, se, tol=2e-5 if loose else 3e-6)
    assert np.abs(se[idx][:, 3:] - so[:, 3:]).max() <= (1e-3 if loose else 1e-4), label
    assert sims[0].stats().dt == sims[1].stats().dt
    assert abs(sims[0].stats().dt - osim.dt) <= 1e-4 * osim.dt, label


@pytest.mark.timeout(300)
@pytest.mark.parametrize("v0,dt_default", [((0.3, -1.0, 0.2), 1e-4), ((1.0, -10.0, 0.5), 1e-3)], ids=["dt_default_binds", "cfl_binds"])
def test_mgsp_two_shards_resume(oracle, cuda_lib, v0, dt_default):
    scene = scenes.small_cube(v0=v0)
    osim = scenes.build_oracle(oracle, scene, dt=dt_default)
    old = [mgsp.build_rank_sim(mgsp.partition_scene(scene, r, 2), r, 2, dt_default, 4000, scenes.apply_material) for r in range(2)]
    ptrs = [s.mgsp_inbox() for s in old]
    for s in old:
        s.mgsp_set_peers(ptrs)
    _threads(lambda s: s.initial_setup(), old)
    for s in old:
        s.step(8)
    for s in old:
        s.sync()
    blobs = [s.save_checkpoint() for s in old]
    assert [checkpoint.info(b)["mgsp_rank"] for b in blobs] == [0, 1]
    for s in old:   # one more sub-step of the uninterrupted pair: its dt comes from the max predicted at the checkpoint
        s.step(1)
    for s in old:
        s.sync()
    dt_next = old[0].stats().dt
    new = [GmpmSimulator.from_checkpoint(b) for b in blobs]
    ptrs = [s.mgsp_inbox() for s in new]
    for s in new:
        s.mgsp_set_peers(ptrs)
    for s in new:   # stage every rank's state first (allocations), then the concurrent set-up that talks to the peer
        s.restore(blobs[s.mgsp_rank], setup=False)
    _threads(lambda s: s.initial_setup(), new)
    osim.step(8)
    _check_mgsp(osim, new, "at the checkpoint", dt_default)
    for s in new:
        s.step(1)
    for s in new:
        s.sync()
    assert new[0].stats().dt == dt_next and new[1].stats().dt == dt_next   # the predicted max is recomputed bit for bit
    for s in new:
        s.step(7)
    for s in new:
        s.sync()
    osim.step(8)
    _check_mgsp(osim, new, "8 sub-steps after the resume", dt_default)
    for s in new + old:
        s.close()


def _err(fn):
    with pytest.raises(CB200Error) as e:
        fn()
    return str(e.value)


def test_rejections_leave_a_usable_simulator(cuda_lib):
    scene = scenes.small_cube()
    esim = scenes.build_engine(scene)
    esim.step(7)
    blob = esim.save_checkpoint()
    inf = checkpoint.info(blob)

    def fresh_setup_works(sim):
        mid = sim.init_model(scene["models"][0]["material"], scene["models"][0]["pos"], scene["models"][0]["v0"])
        scenes.apply_material(sim, mid, scene["models"][0]["material"], 1.0 / 64, False)
        sim.initial_setup()
        sim.step(2)
        assert sim.stats().error == 0
    for kw in (dict(config=Config(domain_bits=6, cfl=0.4)), dict(config=Config(domain_bits=6, boundary=3)), dict(dt=2e-4), dict(fps=24)):
        s = GmpmSimulator.from_checkpoint(blob, **kw)
        assert "CUDA error 1 " in _err(lambda: s.restore(blob))     # cudaErrorInvalidValue
        fresh_setup_works(s)
        s.close()
    s = GmpmSimulator.from_checkpoint(blob, mgsp_world=2, mgsp_rank=0, auto_grow=False)
    assert "CUDA error 1 " in _err(lambda: s.restore(blob))
    s.close()
    s = GmpmSimulator.from_checkpoint(blob, max_blocks=inf["exterior_block_count"] - 1)
    assert "CUDA error 2 " in _err(lambda: s.restore(blob))          # cudaErrorMemoryAllocation
    s.reserve(4000)
    s.restore(blob)
    _assert_round_trip(esim, s, 1)
    s.close()
    s = GmpmSimulator.from_checkpoint(blob)
    _err(lambda: s.checkpoint_begin())                                # not set up
    _err(lambda: s.checkpoint_end())                                  # nothing begun
    fresh_setup_works(s)
    _err(lambda: s.restore(blob))                                     # has models
    s.close()
    # one key moved to an in-domain block the saved particles do not rebuild: an error return, no fault
    bad = blob.copy()
    keys = bad[inf["keys_offset"]: inf["keys_offset"] + inf["keys_bytes"]].view("<i4").reshape(-1, 3)
    keys[inf["neighbor_block_count"] - 1] = (1, 1, 1)
    s = GmpmSimulator.from_checkpoint(bad)
    _err(lambda: s.restore(bad))
    s.close()
    # restored into a larger capacity with auto_grow, then grown again: still the uninterrupted run
    s = _restored(blob, max_blocks=6000, auto_grow=True)
    s.step(3)
    s.reserve(9000)
    s.step(5)
    esim.step(8)
    _compare_state(esim, s, 1, "larger capacity + reserve after a resume")
    assert s.capacity()[0] == 9000
    s.close()
    esim.close()


@pytest.mark.timeout(900)
def test_spheres5m_resume(cuda_lib):
    scene, _ = scenes.workload("spheres5m")
    mb = scenes.max_blocks_for(scene)
    whole = scenes.build_engine(scene, max_blocks=mb)
    whole.step(20)
    blob = whole.save_checkpoint()
    r = _restored(blob)
    _assert_round_trip(whole, r, 2)
    whole.step(20)
    r.step(20)
    _compare_with_live_oracle(whole, r, "spheres5m: 20 + 20 sub-steps vs uninterrupted")
    r.close()
    whole.close()
