"""CPU tests of the boundary impulse report (DESIGN.md section 2.13): the C ABI's exports and constant, every validation of the
new entries (answered before any device work), the scene runner's --forces handling and its MGSP refusal, and the float64
reference (ref64_forces.boundary_impulses) against ref64's own grid update and against impulses worked out by hand."""
import ctypes as C
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import ref64
import ref64_cases as S
import ref64_forces as RF
from claymore_b200 import _capi, objects, scene
from claymore_b200._capi import Config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "claymore_b200.h")
ENTRIES = ("cb200_update_grid_velocity_query_max_forces", "cb200_sim_set_force_report", "cb200_sim_collision_forces")


def test_constant_matches_header(tmp_path):
    gcc = shutil.which("gcc") or shutil.which("cc")
    if gcc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "c.c"
    src.write_text('#include <stdio.h>\n#include "claymore_b200.h"\nint main(void) { printf("%d %d %zu\\n", CB200_FORCE_COMPONENTS, '
                   'CB200_MAX_COLLISION_OBJECTS, sizeof(double)); return 0; }\n')
    exe = tmp_path / "c"
    subprocess.check_call([gcc, "-std=c99", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    out = subprocess.check_output([str(exe)], text=True).split()
    assert out == [str(_capi.FORCE_COMPONENTS), str(_capi.MAX_COLLISION_OBJECTS), "8"]


def test_exports_bound():
    import claymore_b200 as cb
    cb.build_library()
    lib = C.CDLL(cb.lib_path())
    hdr = open(HEADER).read()
    for n in ENTRIES:
        assert hasattr(lib, n), n
        assert n in _capi._SIGNATURES, n
        m = re.search(rf"CB200_API int {n}\(([^)]*)\);", hdr)
        assert m, n
        assert len(m.group(1).split(",")) == len(_capi._SIGNATURES[n]), n


def test_kernel_entry_validates_before_any_launch():
    """block_count 0: an entry that let a bad argument through would return 0 without a launch"""
    import claymore_b200 as cb
    L = cb.lib()
    cfg = Config(domain_bits=6)
    imp = np.zeros((1 + _capi.MAX_COLLISION_OBJECTS) * 6, np.float64)
    ptr = C.c_void_p(imp.ctypes.data)
    good = (_capi.CollisionObject * 1)(objects.box((0.1, 0.1, 0.1), (0.9, 0.2, 0.9)))
    bad = objects.sphere((0.5, 0.5, 0.5), 0.1)
    bad.b[0] = -1.0
    args = lambda objs, n, ls, nls, impulses: (C.byref(cfg), 0, None, _capi.Partition(), 1e-4, None, objs, n, ls, nls, 0.0, None, impulses, None)  # noqa: E731
    assert L.cb200_update_grid_velocity_query_max_forces(*args(good, 1, None, 0, ptr)) == 0
    assert L.cb200_update_grid_velocity_query_max_forces(*args(good, 1, None, 0, None)) != 0                       # no impulses
    assert L.cb200_update_grid_velocity_query_max_forces(*args((_capi.CollisionObject * 1)(bad), 1, None, 0, ptr)) != 0
    assert L.cb200_update_grid_velocity_query_max_forces(*args(good, _capi.MAX_COLLISION_OBJECTS + 1, None, 0, ptr)) != 0
    assert L.cb200_update_grid_velocity_query_max_forces(*args(good, 1, None, -1, ptr)) != 0                       # lattice count
    col = _capi.Collider()
    col.type, col.scale = 0, 0.0                                                                                     # scale 0: invalid
    assert L.cb200_update_grid_velocity_query_max_forces(C.byref(cfg), 0, None, _capi.Partition(), 1e-4, C.byref(col), good, 1, None, 0, 0.0, None,
                                                         ptr, None) != 0
    assert not imp.any()


def test_sim_entries_reject_null_simulator():
    import claymore_b200 as cb
    L = cb.lib()
    out = np.zeros(17 * 6, np.float64)
    n, el = C.c_int(-7), C.c_double(-7.0)
    assert L.cb200_sim_set_force_report(None, 1) != 0
    assert L.cb200_sim_collision_forces(None, C.c_void_p(out.ctypes.data), 17, C.byref(n), C.byref(el)) != 0
    assert (n.value, el.value) == (-7, -7.0)


# ---- the scene runner --------------------------------------------------------------------------------------------------------
def test_forces_flag_parses():
    import claymore_b200.__main__ as M
    with pytest.raises(SystemExit):
        M.main(["--forces"])    # -f is required


def test_forces_refused_in_mgsp_mode():
    doc = {"simulation": {"frames": 1}, "models": [], "boundaries": [{"shape": "box", "offset": [0.1, 0.1, 0.1], "span": [0.8, 0.1, 0.8]}]}
    with pytest.raises(ValueError, match="MGSP"):
        scene.parse_scene(doc, forces=True, mgsp_world=2, mgsp_rank=0)


def test_force_bodies_follow_the_document():
    doc = {"collider": {"file": "x.sdf"}, "boundaries": [{"shape": "box"}, {"shape": "sphere"}, {"shape": "levelset"}]}
    assert scene.force_bodies(doc) == ["collider", "box", "sphere", "levelset"]
    assert scene.force_bodies({"boundaries": [{"shape": "plane"}]}) == ["none", "plane"]


def test_force_recorder_writes_and_appends(tmp_path):
    class Fake:
        force_bodies = ["none", "box"]

        def __init__(self):
            self.t = 0.0

        def collision_forces(self):
            self.t += 0.5
            return 0.5, np.array([[0.0] * 6, [1.0, -2.0, 0.5, 0.0, 0.25, 0.0]])

        def sim_time(self):
            return self.t

    path = str(tmp_path / "forces.csv")
    sim = Fake()
    on_frame, f = scene.force_recorder(sim, path)
    on_frame(sim, 1)
    f.close()
    on_frame, f = scene.force_recorder(sim, path, append=True)
    on_frame(sim, 2)
    f.close()
    rows = open(path).read().strip().split("\n")
    assert rows[0].split(",") == list(scene.FORCE_COLUMNS)
    assert len(rows) == 5
    r = rows[2].split(",")
    assert r[:4] == ["1", "0.5", "1", "box"] and [float(x) for x in r[4:]] == [2.0, -4.0, 1.0, 0.0, 0.5, 0.0]
    assert rows[4].split(",")[0] == "2"
    on_frame, f = scene.force_recorder(sim, path)    # a fresh run truncates
    f.close()
    assert open(path).read().strip().split("\n") == [",".join(scene.FORCE_COLUMNS)]


# ---- the float64 reference ----------------------------------------------------------------------------------------------------
def _one_block(cfg, m, v, key=(4, 4, 4)):
    grid = np.zeros((1, 4, 64), np.float32)
    grid[0, 0] = m
    grid[0, 1:] = (np.asarray(v, np.float32)[:, None] * m).astype(np.float32)
    return np.array([key], np.int32), grid


def test_reference_sticky_box_takes_the_momentum():
    """A static sticky box over a whole block: every node's velocity goes to 0, so J = sum m v_in and L = sum (p - b) x m v_in."""
    cfg = Config(domain_bits=6, boundary=2, gravity=-9.8)
    dx = 1.0 / 64
    keys, grid = _one_block(cfg, 0.5, (1.0, -2.0, 0.25))
    box = objects.box((0.0, 0.0, 0.0), (1.0, 1.0, 1.0), type="sticky", trans=(0.3, 0.2, 0.1))
    r = RF.boundary_impulses(cfg, keys, grid, 1e-3, None, 0.0, [box])
    vin = np.array([1.0, -2.0 + np.float32(-9.8) * 1e-3, 0.25])
    nodes = keys[0] * 4 + ref64._CELLS
    assert np.allclose(r["J"][1], 64 * 0.5 * vin, rtol=1e-6)
    assert np.allclose(r["L"][1], np.cross(nodes * dx - np.float32([0.3, 0.2, 0.1]), 0.5 * vin).sum(0), rtol=1e-6, atol=1e-6)
    assert not r["J"][0].any() and not r["L"][0].any()


def test_reference_chain_ends_where_ref64_does():
    """Summed over the bodies, J is the momentum the whole chain removed: ref64.grid_update's velocities before and after."""
    case = S.OBJECT_CASES["obj_collider_plus_two"]
    cfg = S.config(case)
    rng = np.random.default_rng(3)
    keys = np.array([[k, j, i] for k in range(5, 10) for j in range(3, 8) for i in range(5, 9)], np.int32)
    m = rng.uniform(0.1, 1.0, (len(keys), 64))
    v = rng.normal(0.0, 2.0, (len(keys), 3, 64))
    grid = np.concatenate([m[:, None], m[:, None] * v], 1).astype(np.float32)
    objs = S.object_structs(case)
    col = S.ref_collider(case)
    t = 0.37
    r = RF.boundary_impulses(cfg, keys, grid, 1e-4, col, t, objs)
    has, mm, v0, _ = RF.pre_chain_velocity(cfg, keys, grid, 1e-4)
    v1 = ref64.grid_update(cfg, keys, grid, 1e-4, col, t, objs)[0]
    want = (mm[:, None] * np.where(has[:, None], v0 - v1, 0.0)).sum((0, 2))
    assert np.allclose(r["J"].sum(0), want, rtol=1e-12, atol=1e-12 * np.abs(want).max())
    assert (np.abs(r["J"]).sum(1) > 0).sum() >= 2, "the case must load at least two bodies"
    assert (r["bJ"] >= 0).all() and (r["bL"] >= 0).all()


def test_scene_file_forces_option_writes_nothing_without_gpu(tmp_path):
    """--forces with a scene whose document is refused fails before any file is created"""
    import claymore_b200.__main__ as M
    p = tmp_path / "s.json"
    p.write_text(json.dumps({"models": [{"constitutive": "nope", "type": "particles"}]}))
    with pytest.raises(ValueError):
        M.main(["-f", str(p), "--out", str(tmp_path), "--forces"])
    assert not (tmp_path / "forces.csv").exists()
