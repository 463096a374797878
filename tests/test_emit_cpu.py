"""CPU tests of the emission interface: the exported entries and the header's flag, the scene's "emit" schedule, and every "emit"
validation error, raised before a simulator exists."""
import ctypes as C
import os
import re

import pytest

from claymore_b200 import _capi, scene
from claymore_b200._capi import SdfHeader, SdfSampling

HEADER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "include", "claymore_b200.h")


def test_entries_are_exported_with_the_declared_signatures():
    sig = _capi._SIGNATURES
    assert sig["cb200_sim_add_particles"] == [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_uint, C.POINTER(C.c_int)]
    assert sig["cb200_sim_add_particles_sdf"] == [C.c_void_p, C.c_int, C.POINTER(SdfHeader), C.c_void_p, C.POINTER(SdfSampling), C.c_void_p, C.c_uint,
                                                  C.POINTER(C.c_int)]
    with open(HEADER) as f:
        h = re.sub(r"\s+", " ", f.read())
    assert "CB200_API int cb200_sim_add_particles(cb200_sim* sim, int model, const float* positions_host, int n, const float* v0, unsigned flags, int* n_added);" in h
    assert ("CB200_API int cb200_sim_add_particles_sdf(cb200_sim* sim, int model, const cb200_sdf_header* header, const float* phi_host, "
            "const cb200_sdf_sampling* sampling, const float* v0, unsigned flags, int* n_added);") in h
    m = re.search(r"#define CB200_EMIT_EMPTY_CELLS (\w+) /\* (.*?) \*/", h)
    assert m and int(m.group(1).rstrip("u"), 0) == _capi.EMIT_EMPTY_CELLS == 1 and "cell" in m.group(2)
    lib = _capi.lib_path()
    if os.path.exists(lib):   # built: the symbols are there (nothing is called)
        L = C.CDLL(lib)
        assert hasattr(L, "cb200_sim_add_particles") and hasattr(L, "cb200_sim_add_particles_sdf")


def _doc(emit, frames=10, **model):
    return {"simulation": {"frames": frames}, "models": [dict({"constitutive": "jfluid", "emit": emit}, **model)]}


@pytest.mark.parametrize("emit, frames, want", [
    ({}, 5, [2, 3, 4, 5]),
    ({"start": 3, "every": 3}, 12, [3, 6, 9, 12]),
    ({"start": 2, "every": 2, "until": 7}, 12, [2, 4, 6]),
    ({"start": 4, "until": 4}, 12, [4]),
    ({"start": 8, "until": 20}, 10, [8, 9, 10]),
])
def test_schedule_frames(emit, frames, want):
    assert [f for f, _ in scene.emit_schedule(_doc(emit, frames))[0]] == want


def test_schedule_seeds_and_resume():
    doc = _doc({"start": 2, "every": 2}, 10, seed=5)
    full = scene.emit_schedule(doc)[0]
    assert full == [(2, 7), (4, 9), (6, 11), (8, 13), (10, 15)]
    for F in range(0, 11):   # a run resumed at frame F emits exactly what the uninterrupted run emits after F
        assert scene.emit_schedule(doc, after=F)[0] == [e for e in full if e[0] > F]
    assert scene.emit_schedule({"models": [{"constitutive": "sand"}]}) == {}


@pytest.mark.parametrize("emit", [{"every": 0}, {"every": -1}, {"start": 1}, {"start": 0}, {"start": 5, "until": 4}, {"fill": "half"},
                                  {"rate": 2}, {"start": 2.0}, {"every": True}, "yes"])
def test_bad_emit_raises_before_a_simulator_exists(monkeypatch, emit):
    def no_sim(*a, **k):
        raise AssertionError("a simulator was created")
    monkeypatch.setattr(scene, "GmpmSimulator", type("G", (), {"__init__": no_sim, "DEFAULT_FRAMES": 60, "DEFAULT_DT": 1e-4, "DEFAULT_FPS": 24}))
    with pytest.raises(ValueError):
        scene.parse_scene(_doc(emit))


def test_emit_in_mgsp_mode_raises_before_a_simulator_exists(monkeypatch):
    def no_sim(*a, **k):
        raise AssertionError("a simulator was created")
    monkeypatch.setattr(scene, "GmpmSimulator", type("G", (), {"__init__": no_sim, "DEFAULT_FRAMES": 60, "DEFAULT_DT": 1e-4, "DEFAULT_FPS": 24}))
    with pytest.raises(ValueError, match="MGSP"):
        scene.parse_scene(_doc({}), mgsp_world=2, mgsp_rank=0)


def test_until_defaults_to_the_last_frame_even_before_start():
    assert scene.emit_schedule(_doc({}, frames=1)) == {0: []}
    assert scene.emit_schedule(_doc({"start": 5}, frames=3)) == {0: []}


def test_resume_reads_emit_sources_before_a_simulator_exists(monkeypatch, tmp_path):
    def no_sim(*a, **k):
        raise AssertionError("a simulator was created")
    monkeypatch.setattr(scene, "GmpmSimulator", type("G", (), {"__init__": no_sim, "DEFAULT_FRAMES": 60, "DEFAULT_DT": 1e-4, "DEFAULT_FPS": 24}))
    monkeypatch.setattr(scene, "_check_resume", lambda doc, cfg, resume: {"max_blocks": 100})
    doc = _doc({}, file=str(tmp_path / "missing.bin"))
    with pytest.raises(FileNotFoundError):
        scene.parse_scene(doc, resume="ckpt")
