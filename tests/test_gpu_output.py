"""GPU tests of the per-frame .bgeo output: the gather kernel and the step driver's frame_output / frame_output_wait, the writer thread,
GmpmSimulator.write_frame / wait_output / main_loop(output=...) and the scene runner.

What a file must hold, for one simulator state: positions equal bit for bit, row for row, to the position columns of that model's
section in a checkpoint of the same state; J equals the fluid's J exactly and det F of the checkpoint rows within 1e-5 (float32 cofactor
expansion against a float64 determinant, F near the identity); v equals a float64 numpy G2P over sim.grid() / sim.active_keys() within
2e-6 of max |v| + 1e-7 (float32 weights and a 27-term float32 sum on the device).
"""
import ctypes as C
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

import scenes
from claymore_b200 import bgeo, checkpoint, mgsp
from claymore_b200._capi import CB200Error, Config
from claymore_b200.simulator import GmpmSimulator

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _frame(sim, directory, frame=0, attributes=("v", "J")):
    paths = sim.write_frame(str(directory), frame, attributes)
    sim.wait_output()
    return [bgeo.read(p) for p in paths]


def _rows(blob):
    return checkpoint.read(blob)["states"]


def _g2p(sim, pos):
    """float64 G2P of grid[0]'s node velocities (mv / m, 0 where m = 0) with the engine's base cell and weights"""
    dxi = np.float32(1 << sim.cfg.domain_bits)
    dx = np.float32(1.0) / dxi
    keys, grid = sim.active_keys(), sim.grid()
    keys = keys[: len(grid)].astype(np.int64)
    h = scenes.key_hash(keys)
    order = np.argsort(h)
    hs = h[order]
    base = (np.floor(np.abs(pos * dxi) + np.float32(0.5)) * np.sign(pos)).astype(np.int64) - 1   # roundf: half away from zero
    lp = (pos - base.astype(np.float32) * dx).astype(np.float32)
    d = (lp * dxi).astype(np.float64)
    w = np.stack([0.5 * (1.5 - d) ** 2, 0.75 - (d - 1.0) ** 2, 0.5 * (d - 0.5) ** 2], axis=2)   # [n, axis, node]
    v = np.zeros((len(pos), 3))
    for i in range(3):
        for j in range(3):
            for k in range(3):
                g = base + np.array([i, j, k])
                kh = scenes.key_hash(g >> 2)
                at = np.clip(np.searchsorted(hs, kh), 0, len(hs) - 1)
                found = hs[at] == kh
                b = order[at]
                cell = (g[:, 0] & 3) * 16 + (g[:, 1] & 3) * 4 + (g[:, 2] & 3)
                m = np.where(found, grid[b, 0, cell], 0.0).astype(np.float64)
                mv = np.where(found[:, None], grid[b, 1:4, cell], 0.0).astype(np.float64)
                vel = np.where(m[:, None] > 0, mv / np.where(m > 0, m, 1.0)[:, None], 0.0)
                v += (w[:, 0, i] * w[:, 1, j] * w[:, 2, k])[:, None] * vel
    return v


def _check_file(sim, f, rows, material, label):
    assert f["position"].shape == (len(rows), 3), label
    assert f["position"].view(np.uint32).tobytes() == np.ascontiguousarray(rows[:, :3]).view(np.uint32).tobytes(), label
    if "J" in f:
        if material == scenes.J_FLUID:
            assert f["J"].tobytes() == np.ascontiguousarray(rows[:, 3]).tobytes(), label
        else:
            det = np.linalg.det(rows[:, 3:12].astype(np.float64).reshape(-1, 3, 3))
            assert np.abs(f["J"] - det).max() <= 1e-5, label
    if "v" in f:
        ref = _g2p(sim, rows[:, :3])
        assert np.abs(f["v"] - ref).max() <= 2e-6 * np.abs(ref).max() + 1e-7, label


@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
@pytest.mark.parametrize("material", [scenes.FIXED_COROTATED, scenes.J_FLUID, scenes.SAND, scenes.NACC])
def test_file_matches_checkpoint_rows_and_grid(cuda_lib, tmp_path, material, use_graph):
    sim = scenes.build_engine(scenes.small_cube(material=material), use_graph=use_graph)
    sim.step(7)
    before = sim.save_checkpoint()
    f = _frame(sim, tmp_path)
    after = sim.save_checkpoint()
    assert before.tobytes() == after.tobytes()           # the output only reads
    _check_file(sim, f[0], _rows(before)[0], material, "after 7 sub-steps")
    # overlap: the frame is gathered, then 5 sub-steps run while it is copied and written
    os.makedirs(tmp_path / "o")
    sim.write_frame(str(tmp_path / "o"), 0, ("v", "J"))
    sim.step(5)
    sim.wait_output()
    g = bgeo.read(str(tmp_path / "o" / "model_id[0]_frame[0].bgeo"))
    for k in f[0]:
        assert g[k].tobytes() == f[0][k].tobytes(), k
    assert sim.stats().steps == 12 and sim.stats().error == 0
    sim.close()


def test_velocity_right_after_setup_is_v0(cuda_lib, tmp_path):
    v0 = (0.3, -1.0, 0.2)
    for material in (scenes.FIXED_COROTATED, scenes.J_FLUID):
        sim = scenes.build_engine(scenes.small_cube(material=material, v0=v0))
        f = _frame(sim, tmp_path, attributes=("v",))[0]
        assert set(f) == {"position", "v"}
        assert np.abs(f["v"] - np.array(v0, np.float32)).max() <= 1e-6
        sim.close()


def test_two_models_and_back_pressure(cuda_lib, tmp_path):
    sim = scenes.build_engine(scenes.two_cubes_colliding(), dt=2e-4)
    sim.step(7)
    a = _rows(sim.save_checkpoint())
    pa = sim.write_frame(str(tmp_path), 1, ("J",))
    sim.step(3)
    b = _rows(sim.save_checkpoint())
    pb = sim.write_frame(str(tmp_path), 2, ("J", "v"))   # the first frame is still in flight: this call waits for it
    sim.wait_output()
    for m in range(2):
        _check_file(sim, bgeo.read(pa[m]), a[m], scenes.FIXED_COROTATED, f"frame 1 model {m}")
        fb = bgeo.read(pb[m])
        assert fb["position"].tobytes() == np.ascontiguousarray(b[m][:, :3]).tobytes()
    sim.close()


def test_positions_only_equal_reference_write_partio(cuda_lib, tmp_path):
    shim_path = os.path.join(ROOT, "oracle", "_ref", "libclaymore_ref_partio.so")
    if not os.path.exists(shim_path):
        pytest.skip("oracle/_ref/libclaymore_ref_partio.so not built")
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import make_ref_bgeo_golden as mk
    shim = mk.load_shim()
    sim = scenes.build_engine(scenes.small_cube(material=scenes.SAND))
    sim.step(9)
    rows = _rows(sim.save_checkpoint())[0]
    path = sim.write_frame(str(tmp_path), 3)[0]
    sim.wait_output()
    ref = str(tmp_path / "ref.bgeo")
    mk.write(shim, ref, np.concatenate([rows[:, :3], np.zeros((len(rows), 4), np.float32)], 1), False, False)
    assert open(path, "rb").read() == open(ref, "rb").read()
    sim.close()


def test_main_loop_writes_the_reference_names_and_resumes(cuda_lib, tmp_path):
    scene = scenes.small_cube()
    sim = GmpmSimulator(dt=1e-4, fps=240, frames=3, config=Config(domain_bits=scene["domain_bits"]), max_blocks=4000)
    m = scene["models"][0]
    scenes.apply_material(sim, sim.init_model(m["material"], m["pos"], m["v0"]), m["material"], 1.0 / (1 << scene["domain_bits"]), False)
    out = tmp_path / "run"
    out.mkdir()
    sim.main_loop(output=str(out), attributes=("v",))
    assert sorted(os.listdir(out)) == [f"model_id[0]_frame[{f}].bgeo" for f in (1, 2, 3)]
    last = bgeo.read(str(out / "model_id[0]_frame[3].bgeo"))
    assert last["position"].tobytes() == np.ascontiguousarray(_rows(sim.save_checkpoint())[0][:, :3]).tobytes()
    sim.close()
    a = scenes.build_engine(scene, fps=240)
    a.advance_frame()
    blob = a.save_checkpoint()
    a.close()
    r = GmpmSimulator.from_checkpoint(blob, frames=3)
    r.restore(blob)
    out2 = tmp_path / "resumed"
    out2.mkdir()
    r.main_loop(output=str(out2))
    assert sorted(os.listdir(out2)) == [f"model_id[0]_frame[{f}].bgeo" for f in (2, 3)]
    r.close()


def test_failed_writes_raise_and_leave_the_simulator_usable(cuda_lib, tmp_path):
    sim = scenes.build_engine(scenes.small_cube())
    sim.step(3)
    missing = tmp_path / "missing"
    sim.write_frame(str(missing), 1)
    with pytest.raises(OSError) as e:
        sim.wait_output()
    assert e.value.filename == str(missing / "model_id[0]_frame[1].bgeo") and e.value.errno == 2
    # the error of a frame is also reported by the next write_frame, which then queues nothing
    sim.write_frame(str(missing), 2)
    with pytest.raises(OSError):
        sim.write_frame(str(tmp_path), 2)
    assert not os.path.exists(tmp_path / "model_id[0]_frame[2].bgeo")
    if os.geteuid() != 0:   # permission bits do not stop root
        ro = tmp_path / "ro"
        ro.mkdir()
        os.chmod(ro, 0o500)
        sim.write_frame(str(ro), 1)
        with pytest.raises(OSError) as e:
            sim.wait_output()
        assert e.value.errno == 13
        assert os.listdir(ro) == []
    # argument checks: unknown bits, a null path, a simulator not set up; each leaves it usable
    L = sim.L
    paths = (C.c_char_p * 1)(str(tmp_path / "x.bgeo").encode())
    assert L.cb200_sim_frame_output(sim.h, paths, 4) == 1
    assert L.cb200_sim_frame_output(sim.h, (C.c_char_p * 1)(None), 0) == 1
    with pytest.raises(ValueError):
        sim.write_frame(str(tmp_path), 1, ("w",))
    fresh = GmpmSimulator(config=sim.cfg)
    with pytest.raises(CB200Error):
        fresh.write_frame(str(tmp_path), 1)
    fresh.close()
    sim.step(2)
    rows = _rows(sim.save_checkpoint())[0]
    f = _frame(sim, tmp_path, 5)[0]
    _check_file(sim, f, rows, scenes.FIXED_COROTATED, "after the failures")
    sim.close()


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


@pytest.mark.timeout(300)
def test_mgsp_two_ranks_write_their_own_rows(cuda_lib, tmp_path):
    scene = scenes.small_cube(v0=(0.3, -1.0, 0.2))
    sims = [mgsp.build_rank_sim(mgsp.partition_scene(scene, r, 2), r, 2, 1e-4, 4000, scenes.apply_material) for r in range(2)]
    ptrs = [s.mgsp_inbox() for s in sims]
    for s in sims:
        s.mgsp_set_peers(ptrs)
    _threads(lambda s: s.initial_setup(), sims)
    for s in sims:
        s.step(8)
    for s in sims:    # no rank has sub-steps in flight when the first output allocates its buffers
        s.sync()
    for s in sims:
        rows = _rows(s.save_checkpoint())[0]
        paths = s.write_frame(str(tmp_path), 4, ("v", "J"))
        s.wait_output()
        assert os.path.basename(paths[0]) == f"model_id[0]_rank[{s.mgsp_rank}]_frame[4].bgeo"
        _check_file(s, bgeo.read(paths[0]), rows, scenes.FIXED_COROTATED, f"rank {s.mgsp_rank}")
    for s in sims:
        s.step(4)
    for s in sims:
        s.sync()
    for s in sims:
        s.close()


@pytest.mark.timeout(900)
def test_spheres5m_positions_equal_checkpoint_rows(cuda_lib, tmp_path):
    scene, _ = scenes.workload("spheres5m")
    sim = scenes.build_engine(scene, max_blocks=scenes.max_blocks_for(scene))
    sim.step(20)
    rows = _rows(sim.save_checkpoint())
    paths = sim.write_frame(str(tmp_path), 1, ("J",))
    sim.step(5)
    sim.wait_output()
    for m, p in enumerate(paths):
        f = bgeo.read(p)
        assert f["position"].tobytes() == np.ascontiguousarray(rows[m][:, :3]).tobytes(), m
        assert np.abs(f["J"] - np.linalg.det(rows[m][:, 3:12].astype(np.float64).reshape(-1, 3, 3))).max() <= 1e-5
    sim.close()


def test_scene_runner_cli(cuda_lib, tmp_path):
    doc = {"simulation": {"fps": 240, "frames": 2, "default_dt": 1e-4},
           "models": [{"type": "particles", "constitutive": "jfluid", "file": "box", "offset": [0.3, 0.3, 0.3], "span": [0.1, 0.1, 0.1],
                       "velocity": [0.0, -0.5, 0.0], "rho": 1000, "volume": 1.9e-6, "bulk_modulus": 4e4, "gamma": 7.15, "viscosity": 0.01}]}
    (tmp_path / "scene.json").write_text(json.dumps(doc))
    out = tmp_path / "out"
    out.mkdir()
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-m", "claymore_b200", "-f", str(tmp_path / "scene.json"), "--out", str(out), "--attributes", "v,J"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:]
    assert sorted(os.listdir(out)) == ["model_id[0]_frame[1].bgeo", "model_id[0]_frame[2].bgeo"]
    f = bgeo.read(str(out / "model_id[0]_frame[2].bgeo"))
    assert set(f) == {"position", "v", "J"} and len(f["position"]) > 0 and np.isfinite(f["v"]).all()
