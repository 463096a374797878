"""CPU tests of the analytic collision objects (DESIGN.md section 2.9): the C ABI's struct and exports, the Python constructors'
and the scene parser's validation, and the float64 reference (ref64.object_query) against the level-set collider's fields."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import ref64
from claymore_b200 import _capi, levelset, objects, scene
from claymore_b200._capi import Config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "claymore_b200.h")


def test_struct_layout_matches_gcc(tmp_path):
    gcc = shutil.which("gcc") or shutil.which("cc")
    if gcc is None:
        pytest.skip("no C compiler")
    fields = [f for f, _ in _capi.CollisionObject._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "claymore_b200.h"\nint main(void) {\n'
                   + f'printf("%zu\\n", sizeof(cb200_collision_object));\n'
                   + "".join(f'printf("%zu\\n", offsetof(cb200_collision_object, {f}));\n' for f in fields)
                   + 'printf("%d %d %d %d %d\\n", CB200_SHAPE_PLANE, CB200_SHAPE_BOX, CB200_SHAPE_SPHERE, CB200_SHAPE_CYLINDER, CB200_MAX_COLLISION_OBJECTS);\nreturn 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.check_call([gcc, "-std=c99", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    out = subprocess.check_output([str(exe)], text=True).split("\n")
    assert int(out[0]) == C.sizeof(_capi.CollisionObject)
    for i, f in enumerate(fields):
        assert int(out[1 + i]) == getattr(_capi.CollisionObject, f).offset, f
    assert out[1 + len(fields)].split() == [str(v) for v in (_capi.SHAPE_PLANE, _capi.SHAPE_BOX, _capi.SHAPE_SPHERE, _capi.SHAPE_CYLINDER,
                                                               _capi.MAX_COLLISION_OBJECTS)]


def test_exports_bound():
    import claymore_b200 as cb
    cb.build_library()
    lib = C.CDLL(cb.lib_path())
    hdr = open(HEADER).read()
    for n in ("cb200_update_grid_velocity_query_max_objects", "cb200_sim_set_collision_objects"):
        assert hasattr(lib, n), n
        assert n in _capi._SIGNATURES, n
        assert re.search(rf"CB200_API int {n}\(", hdr), n


def test_kernel_entry_rejects_bad_objects_before_any_launch():
    """The kernel-level entry validates on the host before anything else (block_count 0: an entry that let the list through
    would return 0 without a launch)."""
    import claymore_b200 as cb
    L = cb.lib()
    cfg = Config(domain_bits=6)
    bad = objects.sphere((0.5, 0.5, 0.5), 0.1)
    bad.b[0] = -1.0
    arr = (_capi.CollisionObject * 1)(bad)
    assert L.cb200_update_grid_velocity_query_max_objects(C.byref(cfg), 0, None, _capi.Partition(), 1e-4, None, arr, 1, 0.0, None, None) != 0
    assert L.cb200_update_grid_velocity_query_max_objects(C.byref(cfg), 0, None, _capi.Partition(), 1e-4, None, arr, 17, 0.0, None, None) != 0
    assert L.cb200_update_grid_velocity_query_max_objects(C.byref(cfg), 0, None, _capi.Partition(), 1e-4, None, arr, -1, 0.0, None, None) != 0
    assert L.cb200_sim_set_collision_objects(None, arr, 0) != 0


BAD = [
    (lambda: objects.plane((0, 0, 0), (0, 0, 0)), "normal"),
    (lambda: objects.box((0, 0.5, 0), (1, 0.4, 1)), "lo <= hi"),
    (lambda: objects.sphere((0.5, 0.5, 0.5), 0.0), "radius"),
    (lambda: objects.cylinder((0.5, 0.5, 0.5), 0.1, -0.1), "half height"),
    (lambda: objects.cylinder((0.5, 0.5, 0.5), -0.1, 0.1), "radius"),
    (lambda: objects.box((0, 0, 0), (1, 1, 1), scale=0.0), "scale"),
    (lambda: objects.box((0, 0, 0), (1, 1, 1), type="bouncy"), "boundary type"),
    (lambda: objects.box((0, 0, 0), (1, 1, 1), type=7), "boundary type"),
    (lambda: objects.sphere((0.5, np.nan, 0.5), 0.1), "finite"),
    (lambda: objects.sphere((0.5, 0.5, 0.5), 0.1, trans_vel=(np.inf, 0, 0)), "finite"),
    (lambda: objects.array([objects.sphere((0.5, 0.5, 0.5), 0.1)] * 17), "at most"),
]


@pytest.mark.parametrize("make,msg", BAD, ids=[f"bad{i}" for i in range(len(BAD))])
def test_constructor_validation(make, msg):
    with pytest.raises(ValueError, match=msg):
        make()


def test_plane_normal_is_normalised_in_double():
    o = objects.plane((0.5, 0.3, 0.5), (0.3, -1.0, 0.2))
    u = np.array([0.3, -1.0, 0.2]) / np.linalg.norm([0.3, -1.0, 0.2])
    assert np.array_equal(np.asarray(o.b, np.float32), u.astype(np.float32))


def _doc(boundaries):
    return {"models": [{"constitutive": "jfluid", "file": "box", "offset": [0.3, 0.3, 0.3], "span": [0.1, 0.1, 0.1], "rho": 1000,
                        "volume": 1e-6, "bulk_modulus": 1e4, "gamma": 7, "viscosity": 0}], "boundaries": boundaries}


SCENE_BAD = [
    ([{"shape": "torus"}], "unknown shape"),
    ([{"shape": "box", "colour": "red"}], "unknown keys"),
    ([{"shape": "box", "type": "bouncy"}], "boundary type"),
    ([{"shape": "box", "span": [1, -1, 1]}], "lo <= hi"),
    ([{"shape": "sphere", "span": [0, 1, 1]}], "radius"),
    ([{"shape": "cylinder", "span": [1, 0, 1]}], "half height"),
    ([{"shape": "plane", "normal": [0, 0, 0]}], "normal"),
    ([{"shape": "box", "scale": 0}], "scale"),
    ([{"shape": "box", "velocity": [1, 2]}], "components"),
    ([{"shape": "box", "friction": float("nan")}], "finite"),
    ([{"shape": "box"}] * 17, "at most"),
    ({"shape": "box"}, "list"),
    (["box"], "must be an object"),
]


@pytest.mark.parametrize("bs,msg", SCENE_BAD, ids=[f"scene_bad{i}" for i in range(len(SCENE_BAD))])
def test_scene_boundaries_rejected_before_device_work(bs, msg, monkeypatch):
    def no_device(*a, **k):
        raise AssertionError("a simulator was created for an invalid scene")
    monkeypatch.setattr(scene.GmpmSimulator, "__init__", no_device)
    with pytest.raises(ValueError, match=msg):
        scene.parse_scene(_doc(bs))


def test_scene_placement_conventions():
    bs = scene.boundaries({"boundaries": [
        {"shape": "box", "offset": [0.1, 0.1, 0.1], "span": [0.8, 0.2, 0.8], "type": "slip", "friction": 0.0},
        {"shape": "sphere", "offset": [0.2, 0.3, 0.4], "span": [0.2, 0.3, 0.4]},
        {"shape": "plane", "offset": [0.5, 0.2, 0.5], "normal": [0, 2, 0], "velocity": [0.1, 0, 0]},
        {"shape": "cylinder", "offset": [0.4, 0.2, 0.3], "span": [0.2, 0.4, 0.3], "omega": [0, 1, 0], "dsdt": 0.1, "scale": 1.2}]})
    f = lambda v: list(np.float32(v))   # noqa: E731
    assert (bs[0].shape, list(bs[0].a), list(bs[0].b), bs[0].type) == (_capi.SHAPE_BOX, f([0.1, 0.1, 0.1]), f([0.9, 0.3, 0.9]), _capi.SLIP)
    assert list(bs[1].a) == f([0.3, 0.45, 0.6]) and bs[1].b[0] == np.float32(0.1)
    assert list(bs[2].b) == [0, 1, 0] and list(bs[2].trans_vel) == f([0.1, 0, 0])
    assert list(bs[3].a) == f([0.5, 0.4, 0.45]) and (bs[3].b[0], bs[3].b[1]) == (np.float32(0.1), np.float32(0.2))
    assert (bs[3].dsdt, bs[3].scale) == (np.float32(0.1), np.float32(1.2)) and list(bs[3].omega) == [0, 1, 0]
    assert all(b.friction == np.float32(0.3) for b in bs[1:]) and all(b.type == _capi.STICKY for b in bs[1:])


# ---- the reference against the level-set collider's fields ---------------------------------------------------------------------
def _surface_gap(p, x):
    """float64 distances at the material-space points x[n, 3] of the box, sphere or plane p (ref64.object_params): |phi| to the
    surface, and inside the shape the gap to its nearest normal switch (a box's face tie or centre, a sphere's centre)"""
    sw = np.full(len(x), np.inf)
    if p["shape"] == ref64.PLANE:
        return np.abs((x - p["a"]) @ p["b"]), sw
    if p["shape"] == ref64.BOX:
        ql, qh = p["a"] - x, x - p["b"]
        q = np.maximum(ql, qh)
        srt, i, axis = np.sort(q, 1), np.arange(len(x)), np.argmax(q, 1)
        phi, sw = srt[:, 2], np.minimum(srt[:, 2] - srt[:, 1], np.abs(ql[i, axis] - qh[i, axis]))
    else:
        sw = np.sqrt(((x - p["a"]) ** 2).sum(1))
        phi = sw - p["b"][0]
    return np.abs(phi), np.where(phi <= 0, sw, np.inf)


@pytest.mark.parametrize("shape", ["box", "sphere", "plane"])
@pytest.mark.parametrize("typ", [0, 1, 2])
def test_reference_matches_levelset_fields(shape, typ):
    """For a static box, sphere and plane the analytic shape's hit test and normal are the ones levelset.box / sphere / plane give
    at every grid node that is not near a surface or a face tie: the shape is written in world space at t = 0."""
    cfg = Config(domain_bits=5)
    N, dx = 4 * cfg.grid_size, cfg.dx
    if shape == "box":
        o, (sdf, grad) = objects.box((0.3, 0.28, 0.33), (0.68, 0.61, 0.7), type=typ), levelset.box(cfg, (0.3, 0.28, 0.33), (0.68, 0.61, 0.7))
    elif shape == "sphere":
        o, (sdf, grad) = objects.sphere((0.52, 0.47, 0.5), 0.21, type=typ), levelset.sphere(cfg, (0.52, 0.47, 0.5), 0.21)
    else:
        o, (sdf, grad) = objects.plane((0.5, 0.55, 0.5), (0.3, -1.0, 0.2), type=typ), levelset.plane(cfg, (0.5, 0.55, 0.5), (0.3, -1.0, 0.2))
    nodes = np.stack(np.meshgrid(*[np.arange(N)] * 3, indexing="ij"), -1).reshape(-1, 3)
    p = ref64.object_params(o)
    x = nodes * dx
    q = ref64.object_query(p, (x, np.zeros_like(x)))
    hit, n = q["hit"], q["on"]
    near = np.minimum(*_surface_gap(p, x)) <= 1e-6
    d = sdf.reshape(-1)
    g = grad.reshape(3, -1).T
    keep = ~near & (np.abs(d) > 1e-5)
    assert keep.sum() > 0.9 * len(nodes)
    assert np.array_equal(hit[keep], d[keep] <= 0)
    inside = keep & hit
    assert inside.sum() > 100
    assert np.allclose(n[inside], g[inside], atol=1e-6)
    rng = np.random.default_rng(typ)
    v = rng.normal(0, 1, (len(nodes), 3))
    out = ref64.object_resolve(cfg, p, 0.0, nodes, v, np.abs(v))["v"]
    assert np.array_equal(out[keep & ~hit], v[keep & ~hit])
    if typ == 0:
        assert (out[inside] == 0).all()


@pytest.mark.parametrize("t", [0.0, 0.37])
@pytest.mark.parametrize("typ", [0, 1, 2])
@pytest.mark.parametrize("shape", ["box", "sphere", "plane"])
def test_velocity_matches_dense_collider_reference(shape, typ, t):
    """Velocities through both paths: an analytic object and the float64 reference of the level-set collider (ref64.collider_resolve)
    on the field levelset makes for the same shape, with the same moving parameters, agree at every node that is not near a
    surface, a face tie or the wall band.  This pins the objects' material space and motion to the collider's."""
    cfg = Config(domain_bits=5, boundary=2)
    N, dx = 4 * cfg.grid_size, cfg.dx
    motion = dict(trans_vel=(0.05, -0.04, 0.03))
    kw = dict(type=typ, friction=0.3, **motion)
    if shape == "box":
        o, (sdf, grad) = objects.box((0.3, 0.28, 0.33), (0.68, 0.61, 0.7), **kw), levelset.box(cfg, (0.3, 0.28, 0.33), (0.68, 0.61, 0.7))
    elif shape == "sphere":
        o, (sdf, grad) = objects.sphere((0.52, 0.47, 0.5), 0.21, **kw), levelset.sphere(cfg, (0.52, 0.47, 0.5), 0.21)
    else:
        o, (sdf, grad) = objects.plane((0.5, 0.55, 0.5), (0.0, 1.0, 0.0), **kw), levelset.plane(cfg, (0.5, 0.55, 0.5), (0.0, 1.0, 0.0))
    col = dict(rot_mat=np.eye(3).reshape(9), trans=(0.0, 0.0, 0.0), trans_vel=motion["trans_vel"], omega=(0.0, 0.0, 0.0), dsdt=0.0, scale=1.0,
               friction=0.3, type=typ)
    rng = np.random.default_rng(typ)
    lo, hi = 4 * cfg.boundary, N - 4 * cfg.boundary
    nodes = np.stack(np.meshgrid(*[np.arange(lo, hi)] * 3, indexing="ij"), -1).reshape(-1, 3)
    v = rng.normal(0, 1, (len(nodes), 3))
    r = ref64.collider_resolve(cfg, col, sdf, grad, np.float32(t), nodes, v, np.zeros_like(v))
    p = ref64.object_params(o)
    ro = ref64.object_resolve(cfg, p, np.float32(t), nodes, v, np.zeros_like(v))
    out, ohit = ro["v"], ro["hit"]
    # the trilinear field is exact only a cell away from the surface and from a box's edges and face ties
    x = nodes * dx - np.float32(t) * np.asarray(motion["trans_vel"], np.float32)
    far = np.minimum(*_surface_gap(p, x)) <= 1.5 * dx
    band = ((x < (lo + 1) * dx) | (x >= (hi - 1) * dx)).any(1)      # the collider reports no hit in its wall band (C1)
    keep = ~ro["near"] & ~r["near"] & ~far & ~band
    if shape == "sphere" and t > 0:   # off the lattice the trilinear gradient of a sphere is not its normal: compare the hit test only
        assert np.array_equal(ohit[keep], r["hit"][keep])
        return
    assert keep.sum() > 300
    assert (r["hit"][keep]).sum() > 100 and (~r["hit"][keep]).sum() > 100
    assert np.allclose(out[keep], r["v"][keep], rtol=1e-5, atol=1e-5)
