"""CPU tests of the removal interface: the exported entries and the header's flag, the scene's "sinks" schedule and its grouping, and
every "sinks" validation error, raised before a simulator exists."""
import ctypes as C
import os
import re

import pytest

from claymore_b200 import _capi, scene
from claymore_b200._capi import CollisionObject

HEADER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "include", "claymore_b200.h")


def test_entries_are_exported_with_the_declared_signatures():
    sig = _capi._SIGNATURES
    assert sig["cb200_sim_remove_particles"] == [C.c_void_p, C.c_uint, C.POINTER(CollisionObject), C.c_int, C.c_uint, C.POINTER(C.c_longlong)]
    assert sig["cb200_sim_remove_rows"] == [C.c_void_p, C.c_int, C.c_void_p, C.c_longlong, C.POINTER(C.c_longlong)]
    with open(HEADER) as f:
        h = re.sub(r"\s+", " ", f.read())
    assert ("CB200_API int cb200_sim_remove_particles(cb200_sim* sim, unsigned model_mask, const cb200_collision_object* regions, int n, "
            "unsigned flags, long long* removed);") in h
    assert "CB200_API int cb200_sim_remove_rows(cb200_sim* sim, int model, const unsigned char* remove_host, long long n, long long* removed);" in h
    m = re.search(r"#define CB200_REMOVE_OUTSIDE (\w+) /\* (.*?) \*/", h)
    assert m and int(m.group(1).rstrip("u"), 0) == _capi.REMOVE_OUTSIDE == 1 and "outside" in m.group(2)
    lib = _capi.lib_path()
    if os.path.exists(lib):   # built: the symbols are there (nothing is called)
        L = C.CDLL(lib)
        assert hasattr(L, "cb200_sim_remove_particles") and hasattr(L, "cb200_sim_remove_rows")


def _doc(sinks, frames=10, n_models=2):
    return {"simulation": {"frames": frames}, "models": [{"constitutive": "jfluid"}] * n_models, "sinks": sinks}


def _box(**kw):
    return dict({"shape": "box", "offset": [0.1, 0.1, 0.1], "span": [0.2, 0.2, 0.2]}, **kw)


@pytest.mark.parametrize("spec, frames, want", [
    ({}, 5, [1, 2, 3, 4, 5]),
    ({"start": 3, "every": 3}, 12, [3, 6, 9, 12]),
    ({"start": 2, "every": 2, "until": 7}, 12, [2, 4, 6]),
    ({"start": 4, "until": 4}, 12, [4]),
    ({"start": 8, "until": 20}, 10, [8, 9, 10]),
    ({"start": 12}, 10, []),
])
def test_schedule_frames(spec, frames, want):
    assert list(scene.sink_schedule(_doc([_box(**spec)], frames))) == want


def test_schedule_after_a_resume_at_every_frame():
    doc = _doc([_box(start=2, every=3), _box(shape="sphere", models=[1]), _box(start=5, until=8, outside=True)], 10)
    full = scene.sink_schedule(doc)
    for F in range(0, 11):   # a run resumed at frame F removes exactly what the uninterrupted run removes after F
        assert scene.sink_schedule(doc, after=F) == {f: g for f, g in full.items() if f > F}
    assert scene.sink_schedule({"models": [{"constitutive": "sand"}]}) == {}


def test_sinks_due_together_with_the_same_models_and_outside_share_a_call():
    doc = _doc([_box(), _box(shape="sphere", models=[1, 0]), _box(models=[1]), _box(outside=True), _box(shape="plane", start=2, every=2),
                _box(models=[0], outside=True)], 4)
    got = scene.sink_schedule(doc)
    assert got[1] == [((0, 1), False, [0, 1]), ((1,), False, [2]), ((0, 1), True, [3]), ((0,), True, [5])]
    assert got[2] == [((0, 1), False, [0, 1, 4]), ((1,), False, [2]), ((0, 1), True, [3]), ((0,), True, [5])]
    assert got[3] == got[1]


def test_a_group_holds_at_most_the_object_limit():
    assert len(scene.sinks(_doc([_box()] * 16))) == 16
    assert len(scene.sinks(_doc([_box(models=[0])] * 16 + [_box(models=[1])] * 16))) == 32   # two groups of 16
    with pytest.raises(ValueError, match="at most 16"):
        scene.sinks(_doc([_box()] * 17))
    assert len(scene.sinks(_doc([_box(start=1, until=1)] * 16 + [_box(start=2)]))) == 17   # never due together


def _no_sim(monkeypatch):
    def no_sim(*a, **k):
        raise AssertionError("a simulator was created")
    monkeypatch.setattr(scene, "GmpmSimulator", type("G", (), {"__init__": no_sim, "DEFAULT_FRAMES": 60, "DEFAULT_DT": 1e-4, "DEFAULT_FPS": 24}))


@pytest.mark.parametrize("sinks", [
    "box", [1], [{"offset": [0, 0, 0]}], [_box(shape="cone")], [_box(type="slip")], [_box(friction=0.1)], [_box(rate=2)],
    [_box(models=[2])], [_box(models=[-1])], [_box(models=[])], [_box(models=0)], [_box(models=[True])], [_box(models=[0.0])],
    [_box(outside=1)], [_box(outside="yes")], [_box(start=0)], [_box(every=0)], [_box(start=5, until=4)], [_box(start=2.0)],
    [_box(every=True)], [_box(until="end")], [_box(span=[1, 1])], [_box(span=[-0.1, 0.1, 0.1])], [_box(shape="sphere", span=[0, 1, 1])],
    [_box(shape="plane", normal=[0, 0, 0])], [_box(scale=0)], [_box(velocity=[float("nan"), 0, 0])], [_box()] * 17,
])
def test_bad_sinks_raise_before_a_simulator_exists(monkeypatch, sinks):
    _no_sim(monkeypatch)
    with pytest.raises(ValueError):
        scene.parse_scene(_doc(sinks))


def test_sinks_in_mgsp_mode_raise_before_a_simulator_exists(monkeypatch):
    _no_sim(monkeypatch)
    with pytest.raises(ValueError, match="MGSP"):
        scene.parse_scene(_doc([_box()]), mgsp_world=2, mgsp_rank=0)


def test_sink_regions_are_placed_as_boundaries_are():
    entry = {"offset": [0.1, 0.2, 0.3], "span": [0.2, 0.3, 0.4], "normal": [0, 0, 1], "velocity": [0.1, 0, 0], "omega": [0, 1, 0], "scale": 2.0,
             "dsdt": 0.5}
    for shape in ("box", "sphere", "plane", "cylinder"):
        a = scene.sinks(_doc([dict(entry, shape=shape, models=[0])]))[0]["object"]
        b = scene.boundaries({"boundaries": [dict(entry, shape=shape)]})[0]
        assert bytes(a) == bytes(b), shape
