"""CPU tests of the level-set collision objects (CB200_SHAPE_LEVELSET, DESIGN.md section 2.11): the C ABI mirror, every rejection
that needs no device, the scene parser's errors (all raised before any simulator exists), and the float64 query of
ref64_levelset against an independent trilinear restatement on sdf_ref's lattices."""
import ctypes as C
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import ref64
import ref64_levelset as RL
import sdf_ref
from claymore_b200 import _capi, objects, scene, sdf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "claymore_b200.h")
INVALID = 1   # cudaErrorInvalidValue

LATTICES = {
    "sphere": lambda: sdf_ref.sphere((16, 16, 16), 0.1, (0.75, 0.75, 0.75), 0.5),
    "torus": lambda: sdf_ref.torus((20, 12, 20), 0.1, (0.95, 0.55, 0.95), 0.6, 0.22),
    "box": lambda: sdf_ref.box((10, 14, 9), 0.2, (0.3, 0.5, 0.35), (1.5, 2.1, 1.2)),
    "plate": lambda: sdf_ref.plate((9, 7, 8), 0.25, 3),
    "dragonish": lambda: sdf_ref.dragonish(),
}


def level_set(name):
    n, h, phi = LATTICES[name]()
    return sdf.parse(sdf_ref.text(n, h, np.asarray(phi, np.float32)))


def test_struct_constants_and_exports(tmp_path):
    gcc = shutil.which("gcc") or shutil.which("cc")
    if gcc is None:
        pytest.skip("no C compiler")
    fields = [f for f, _ in _capi.LevelSetLattice._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "claymore_b200.h"\nint main(void) {\n'
                   + 'printf("%zu\\n", sizeof(cb200_levelset));\n'
                   + "".join(f'printf("%zu\\n", offsetof(cb200_levelset, {f}));\n' for f in fields)
                   + 'printf("%d %d\\n", CB200_SHAPE_LEVELSET, CB200_MAX_COLLISION_LEVELSETS);\nreturn 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.check_call([gcc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    out = subprocess.check_output([str(exe)], text=True).split("\n")
    assert int(out[0]) == C.sizeof(_capi.LevelSetLattice)
    for i, f in enumerate(fields):
        assert int(out[1 + i]) == getattr(_capi.LevelSetLattice, f).offset, f
    assert out[1 + len(fields)].split() == [str(_capi.SHAPE_LEVELSET), str(_capi.MAX_COLLISION_LEVELSETS)]
    lib = _capi.lib()
    hdr = open(HEADER).read()
    for n in ("cb200_levelset_prepare", "cb200_update_grid_velocity_query_max_levelsets", "cb200_sim_add_collision_levelset",
              "cb200_sim_clear_collision_levelsets"):
        assert hasattr(lib, n) and n in _capi._SIGNATURES and re.search(rf"CB200_API int {n}\(", hdr), n


# ---- rejections without a device ---------------------------------------------------------------------------------------------
def _grid_call(objs, lattices, n_lattices=None, entry="levelsets"):
    """the kernel-level entry on a 0-block grid: validation runs, nothing is launched"""
    lib = _capi.lib()
    cfg = _capi.Config(domain_bits=6)
    arr = (_capi.CollisionObject * max(len(objs), 1))(*objs)
    part = _capi.Partition()
    if entry == "objects":
        return lib.cb200_update_grid_velocity_query_max_objects(C.byref(cfg), 0, None, part, 1e-4, None, arr, len(objs), 0.0, None, None)
    lv = (_capi.LevelSetLattice * max(len(lattices), 1))(*lattices)
    n = len(lattices) if n_lattices is None else n_lattices
    return lib.cb200_update_grid_velocity_query_max_levelsets(C.byref(cfg), 0, None, part, 1e-4, None, arr, len(objs), lv, n, 0.0, None, None)


def _raw(index=0.0, c=0.01):
    o = objects.box((0, 0, 0), (1, 1, 1))
    o.shape = _capi.SHAPE_LEVELSET
    o.a[:] = (0.1, 0.1, 0.1)
    o.b[:] = (c, index, 0.0)
    return o


def _view():
    return _capi.LevelSetLattice(0x1000, 4, 5, 6)   # never read: no block is updated


def test_kernel_entry_accepts_a_valid_levelset_and_rejects_every_bad_one():
    assert _grid_call([_raw(0.0)], [_view()]) == 0
    assert _grid_call([_raw(1.0)], [_view(), _view()]) == 0
    assert _grid_call([objects.sphere((0.5, 0.5, 0.5), 0.1)], []) == 0   # no level set, no lattice: the objects path
    bad = {"index not an integer": _raw(0.5), "index negative": _raw(-1.0), "index = count": _raw(1.0), "index NaN": _raw(float("nan")),
           "index inf": _raw(float("inf")), "c = 0": _raw(0.0, 0.0), "c < 0": _raw(0.0, -0.01), "c NaN": _raw(0.0, float("nan"))}
    for what, o in bad.items():
        assert _grid_call([o], [_view()]) == INVALID, what                     # cudaErrorInvalidValue
    assert _grid_call([_raw(0.0)], []) == INVALID, "a level set with no lattice"
    assert _grid_call([_raw(0.0)], [_view()] * 17) == INVALID, "more than CB200_MAX_COLLISION_LEVELSETS lattices"
    assert _grid_call([_raw(0.0)], [_capi.LevelSetLattice(0, 4, 5, 6)]) == INVALID, "a null lattice"
    assert _grid_call([_raw(0.0)], [_capi.LevelSetLattice(0x1000, 1, 5, 6)]) == INVALID, "a dimension below 2"
    assert _grid_call([_raw(0.0)], [_view()], n_lattices=-1) == INVALID


def test_objects_entry_keeps_rejecting_the_levelset_shape():
    assert _grid_call([_raw(0.0)], [], entry="objects") == INVALID
    assert _grid_call([objects.sphere((0.5, 0.5, 0.5), 0.1)], [], entry="objects") == 0


def test_prepare_rejects_bad_headers():
    lib = _capi.lib()
    for dims in ((1, 4, 4), (4, 1, 4), (4, 4, 1), (0, 4, 4), (2048, 2048, 1024)):
        h = _capi.SdfHeader(*dims, (C.c_float * 3)(0, 0, 0), 0.1)
        assert lib.cb200_levelset_prepare(C.byref(h), C.c_void_p(0x1000), C.c_void_p(0x2000), None) == INVALID, dims
    h = _capi.SdfHeader(4, 4, 4, (C.c_float * 3)(0, 0, 0), 0.1)
    assert lib.cb200_levelset_prepare(C.byref(h), None, C.c_void_p(0x2000), None) == INVALID
    assert lib.cb200_levelset_prepare(C.byref(h), C.c_void_p(0x1000), None, None) == INVALID
    assert lib.cb200_levelset_prepare(None, C.c_void_p(0x1000), C.c_void_p(0x2000), None) == INVALID


def test_python_constructor_fits_as_the_sampler_and_validates():
    ls = level_set("torus")
    o = objects.levelset(ls, (0.2, 0.1, 0.3), (0.4, 0.5, 0.6), type="slip", friction=0.2, omega=(0, 1, 0))
    c, lo, _ = sdf.node_box(ls, (0.2, 0.1, 0.3), (0.4, 0.5, 0.6))
    assert o.shape == _capi.SHAPE_LEVELSET and o.levelset is ls
    assert list(o.a) == [float(np.float32(v)) for v in lo] and o.b[0] == np.float32(c) and o.type == _capi.SLIP
    objects.validate(o)
    for span in ((0.0, 1, 1), (1, -1, 1)):
        with pytest.raises(ValueError, match="span"):
            objects.levelset(ls, (0, 0, 0), span)
    for what, bad in {"index": _raw(0.5), "spacing": _raw(0.0, 0.0)}.items():
        with pytest.raises(ValueError, match=what):
            objects.validate(bad)
    with pytest.raises(ValueError, match="index"):
        objects.validate(_raw(2.0), levelsets=2)
    objects.validate(_raw(1.0), levelsets=2)


# ---- scene --------------------------------------------------------------------------------------------------------------------
def _doc(tmp_path, boundaries=(), sinks=()):
    ls = level_set("box")
    (tmp_path / "obstacle.sdf").write_bytes(sdf_ref.text(ls.n, ls.h, ls.phi))
    return {"simulation": {"frames": 3}, "models": [{"constitutive": "jfluid", "file": "box", "offset": [0.4, 0.4, 0.4], "span": [0.1, 0.1, 0.1]}],
            "boundaries": list(boundaries), "sinks": list(sinks)}


def test_scene_levelset_entries_parse_and_share_one_level_set(tmp_path):
    b = {"shape": "levelset", "file": "obstacle.sdf", "offset": [0.7, -0.2, 0.5], "span": [0.6, 0.6, 0.6], "type": "slip", "velocity": [0, 1, 0]}
    doc = _doc(tmp_path, [b], [{"shape": "levelset", "file": str(tmp_path / "obstacle.sdf"), "offset": [0, 0, 0], "span": [0.2, 0.2, 0.2]}])
    cache = {}
    objs = scene.boundaries(doc, str(tmp_path), cache)
    sinks = scene.sinks(doc, str(tmp_path), cache)
    assert objs[0].shape == _capi.SHAPE_LEVELSET and objs[0].type == _capi.SLIP and list(objs[0].trans_vel) == [0, 1, 0]
    assert objs[0].levelset is sinks[0]["object"].levelset, "one file is one level set"
    assert len(cache) == 1


@pytest.mark.parametrize("entry,match", [
    ({"shape": "levelset", "file": "missing.sdf"}, "missing.sdf"),
    ({"shape": "levelset", "file": "obstacle.bin"}, "must name an .sdf"),
    ({"shape": "levelset"}, "must name an .sdf"),
    ({"shape": "levelset", "file": "garbage.sdf"}, "not a valid .sdf"),
    ({"shape": "levelset", "file": "obstacle.sdf", "span": [0.1, 0.0, 0.1]}, "span"),
    ({"shape": "levelset", "file": "obstacle.sdf", "radius": 1}, "unknown keys"),
    ({"shape": "box", "file": "obstacle.sdf"}, "unknown keys"),
    ({"shape": "levelset", "file": "obstacle.sdf", "type": "glue"}, "boundary type|unknown keys"),   # sinks take no type
])
def test_scene_rejects_bad_levelset_entries_before_any_simulator(tmp_path, monkeypatch, entry, match):
    import claymore_b200.simulator as simmod
    (tmp_path / "garbage.sdf").write_text("4 4 4\n0 0 0\n0.1\n1 2 3\n")
    for key in ("boundaries", "sinks"):
        doc = _doc(tmp_path, **{key: [entry]})
        path = tmp_path / "scene.json"
        path.write_text(json.dumps(doc))

        def no_sim(*a, **k):
            raise AssertionError("a simulator was created before the scene was validated")
        monkeypatch.setattr(simmod.GmpmSimulator, "__init__", no_sim)
        with pytest.raises(ValueError, match=match):
            scene.parse_scene(str(path))


def test_scene_obstacle_may_extend_past_the_domain(tmp_path):
    doc = _doc(tmp_path, [{"shape": "levelset", "file": "obstacle.sdf", "offset": [-0.5, 0.8, 0.2], "span": [2.0, 2.0, 2.0]}])
    assert scene.boundaries(doc, str(tmp_path))[0].a[0] == np.float32(-0.5)


# ---- the float64 query --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(LATTICES))
def test_prepare_restatement_is_central_differences(name):
    ls = level_set(name)
    lat = RL.lattice(ls.n, ls.phi)
    g = ls.grid.astype(np.float32)
    assert np.array_equal(lat[..., 0], g)
    assert np.array_equal(lat[1:-1, 1:-1, 1:-1, 1], (np.float32(0.5) * (g[1:-1, 1:-1, 2:] - g[1:-1, 1:-1, :-2])))
    assert np.array_equal(lat[:, :, 0, 1], g[:, :, 1] - g[:, :, 0]) and np.array_equal(lat[:, :, -1, 3 - 2], g[:, :, -1] - g[:, :, -2])
    assert np.array_equal(lat[0, :, :, 3], g[1] - g[0]) and np.array_equal(lat[:, -1, :, 2], g[:, -1] - g[:, -2])


@pytest.mark.parametrize("name", list(LATTICES))
def test_query_matches_an_independent_trilinear_away_from_flagged_points(name):
    """ref64_levelset's hit set equals sdf_ref.trilinear's phi <= 0 and its normal the normalised trilinear g, except at flagged
    points; the flagged share stays small, and both sides of the hit test are reached."""
    ls = level_set(name)
    lat = RL.lattice(ls.n, ls.phi)
    rng = np.random.default_rng(len(name))
    c, a = 0.01, np.array([0.2, 0.1, 0.3])
    dims = np.array(ls.n, np.float64)
    q = rng.uniform(-1.0, dims + 0.5, (20000, 3))
    q[:500] = np.round(q[:500])                                 # on nodes, and on the box faces
    x = (a + q * c).astype(np.float32).astype(np.float64)
    o = dict(shape=RL.LEVELSET, a=a.astype(np.float32).astype(np.float64), b=np.array([np.float32(c), 0.0, 0.0], np.float64))
    r = RL.levelset_query(o, lat, (x, np.zeros_like(x)))
    qq = (x - o["a"]) / o["b"][0]
    inside = np.all((qq >= 0) & (qq <= dims - 1), 1)
    qc = np.clip(qq, 0, dims - 1)
    ref_phi = np.full(len(x), np.inf)
    ref_phi[inside] = sdf_ref.trilinear(ls.n, ls.phi, qc[inside, 0], qc[inside, 1], qc[inside, 2])
    near = r["margin"] <= ref64.NEAR
    assert np.array_equal(r["hit"][~near], (ref_phi <= 0)[~near])
    assert near.mean() < 0.02, f"{near.mean():.3%} flagged"
    assert r["hit"][~near].any() and (~r["hit"][~near] & inside[~near]).any()
    gi = [sdf_ref.trilinear(ls.n, lat[..., k].reshape(-1), qc[inside, 0], qc[inside, 1], qc[inside, 2]) for k in (1, 2, 3)]
    g = np.stack(gi, 1)
    ln = np.linalg.norm(g, axis=1)
    ok = (ln > 0) & r["hit"][inside] & ~near[inside]
    assert np.allclose(r["on"][inside][ok], (g / np.where(ln > 0, ln, 1)[:, None])[ok], atol=1e-9)
