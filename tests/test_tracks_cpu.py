"""CPU tests of collision-object motion tracks (DESIGN.md section 2.14): the C ABI's structs, constants and exports, every rejection
of cb200_track_prepare and of the Python and scene validators, the prepared records against the float64 restatement
(ref64_tracks.prepare), and the float64 evaluation against its own finite differences: c' and omega are the derivatives of c(t) and
R(t) inside segments, before the first key, at keys, after the last key and across a periodic wrap."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import ref64
import ref64_tracks as RT
from claymore_b200 import _capi, objects, scene
from claymore_b200._capi import Config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "claymore_b200.h")
ENTRIES = ("cb200_track_prepare", "cb200_update_grid_velocity_query_max_tracks", "cb200_sim_set_object_track")


@pytest.fixture(autouse=True)
def tracked_reference():
    """ref64's chain and ref64_forces with tracked objects moving on their tracks (ref64_tracks.tracked)"""
    with RT.tracked():
        yield


def _q(axis, angle):
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    return [np.cos(angle / 2)] + list(np.sin(angle / 2) * a)


KEYS = [(0.0, (0.5, 0.5, 0.5), (1, 0, 0, 0)), (0.1, (0.6, 0.5, 0.5), _q((0, 1, 0), 0.6)), (0.25, (0.6, 0.42, 0.45), _q((1, 0.3, 0), 1.0)),
        (0.4, (0.55, 0.45, 0.5), _q((0.2, 1, 0.1), -0.7)), (0.5, (0.5, 0.5, 0.5), (1, 0, 0, 0))]


def test_structs_and_constants_match_header(tmp_path):
    gcc = shutil.which("gcc") or shutil.which("cc")
    if gcc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "c.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "claymore_b200.h"\nint main(void) { printf("%zu %zu %zu %zu %zu %zu %zu %d %d %d %d\\n", '
                   'sizeof(cb200_track_key), sizeof(cb200_track_record), sizeof(cb200_track_span), offsetof(cb200_track_record, rot), '
                   'offsetof(cb200_track_record, tangent), offsetof(cb200_track_record, rotvec), offsetof(cb200_track_key, rot), '
                   'CB200_TRACK_LINEAR, CB200_TRACK_SMOOTH, CB200_TRACK_PERIODIC, CB200_MAX_TRACK_KEYS); return 0; }\n')
    exe = tmp_path / "c"
    subprocess.check_call([gcc, "-std=c99", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    out = subprocess.check_output([str(exe)], text=True).split()
    want = [C.sizeof(_capi.TrackKey), C.sizeof(_capi.TrackRecord), C.sizeof(_capi.TrackSpan), _capi.TrackRecord.rot.offset,
            _capi.TrackRecord.tangent.offset, _capi.TrackRecord.rotvec.offset, _capi.TrackKey.rot.offset,
            _capi.TRACK_LINEAR, _capi.TRACK_SMOOTH, _capi.TRACK_PERIODIC, _capi.MAX_TRACK_KEYS]
    assert out == [str(w) for w in want]
    assert C.sizeof(_capi.TrackRecord) == 64


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


def _raw(keys):
    arr = (_capi.TrackKey * max(len(keys), 1))()
    for i, (t, p, q) in enumerate(keys):
        arr[i].t, arr[i].pos[:], arr[i].rot[:] = t, list(p), [float(x) for x in q]
    return arr


def _prepare(keys, flags):
    import claymore_b200 as cb
    out = (_capi.TrackRecord * max(len(keys), 1))()
    for r in out:
        r.t = -7.0
    e = cb.lib().cb200_track_prepare(_raw(keys), len(keys), flags, out)
    return e, np.frombuffer(out, np.float32).reshape(-1, 16)[: len(keys)]


LOOP = [(0.0, (0.5, 0.5, 0.5), (1, 0, 0, 0)), (0.2, (0.6, 0.5, 0.5), _q((0, 1, 0), 1.0)), (0.4, (0.5, 0.5, 0.5), (1, 0, 0, 0))]
REJECTED = {
    "not_increasing": ([(0.0, (0, 0, 0), (1, 0, 0, 0)), (0.0, (0, 0, 0), (1, 0, 0, 0))], 0),
    "decreasing": ([(0.2, (0, 0, 0), (1, 0, 0, 0)), (0.1, (0, 0, 0), (1, 0, 0, 0))], 0),
    "nan_time": ([(float("nan"), (0, 0, 0), (1, 0, 0, 0))], 0),
    "inf_position": ([(0.0, (0, float("inf"), 0), (1, 0, 0, 0))], 0),
    "nan_rotation": ([(0.0, (0, 0, 0), (1, float("nan"), 0, 0))], 0),
    "zero_quaternion": ([(0.0, (0, 0, 0), (0, 0, 0, 0))], 0),
    "antipodal": ([(0.0, (0, 0, 0), (1, 0, 0, 0)), (0.1, (0, 0, 0), (0, 0, 1, 0))], 0),
    "periodic_position": ([(0.0, (0, 0, 0), (1, 0, 0, 0)), (0.1, (0.1, 0, 0), (1, 0, 0, 0))], _capi.TRACK_PERIODIC),
    "periodic_rotation": ([(0.0, (0, 0, 0), (1, 0, 0, 0)), (0.1, (0, 0, 0), _q((0, 0, 1), 0.5))], _capi.TRACK_PERIODIC),
    "periodic_one_key": ([(0.0, (0, 0, 0), (1, 0, 0, 0))], _capi.TRACK_PERIODIC),
    "too_many": ([(0.001 * i, (0, 0, 0), (1, 0, 0, 0)) for i in range(_capi.MAX_TRACK_KEYS + 1)], 0),
    "no_keys": ([], 0),
}


@pytest.mark.parametrize("name", list(REJECTED))
def test_prepare_rejects(name):
    keys, flags = REJECTED[name]
    e, out = _prepare(keys, flags)
    assert e != 0, name
    assert (out[:, 0] == -7.0).all(), f"{name}: out written on a rejection"
    with pytest.raises(ValueError):
        RT.prepare(keys, flags)
    with pytest.raises(ValueError):
        objects.track(keys, "linear", bool(flags & _capi.TRACK_PERIODIC))


def test_prepare_rejects_unknown_flags_and_nulls():
    import claymore_b200 as cb
    L = cb.lib()
    out = (_capi.TrackRecord * 3)()
    assert L.cb200_track_prepare(_raw(LOOP), 3, 4, out) != 0
    assert L.cb200_track_prepare(None, 3, 0, out) != 0
    assert L.cb200_track_prepare(_raw(LOOP), 3, 0, None) != 0
    with pytest.raises(ValueError):
        objects.track(LOOP, "cubic")


def test_periodic_accepts_quaternion_sign():
    keys = LOOP[:2] + [(0.4, (0.5, 0.5, 0.5), (-1, 0, 0, 0))]
    assert _prepare(keys, _capi.TRACK_PERIODIC)[0] == 0
    objects.track(keys, periodic=True)


@pytest.mark.parametrize("flags", [0, 1, 2, 3])
def test_records_match_float64(flags):
    keys = KEYS if flags & _capi.TRACK_PERIODIC else KEYS[:-1] + [(0.5, (0.52, 0.5, 0.48), _q((0, 0, 1), 2.5))]
    e, got = _prepare(keys, flags)
    assert e == 0
    want = RT.prepare(keys, flags)
    assert np.array_equal(got, want), np.abs(got - want).max()
    # hemisphere alignment: every neighbouring pair on one side, and the slerp ends at the next key
    q = got[:, 4:8].astype(np.float64)
    assert ((q[1:] * q[:-1]).sum(1) > 0).all()
    for k in range(len(keys) - 1):
        r = got[k, 11:14].astype(np.float64)
        th = np.linalg.norm(r)
        end = RT.qmul(q[k], np.concatenate([[np.cos(th / 2)], np.sin(th / 2) * r / th]) if th > 0 else np.array([1.0, 0, 0, 0]))
        assert np.abs(end - q[k + 1]).max() < 1e-6


def test_python_track_matches_prepare():
    tr = objects.track([(t, p, RT.quat_mat(q)) for t, p, q in KEYS], "smooth", periodic=True)   # rotations as matrices
    e, got = _prepare(KEYS, tr.flags)
    want = RT.prepare(tr.keys, tr.flags)
    assert e == 0 and np.abs(got - want).max() < 1e-6


def test_object_track_keyword_rejects_reference_motion():
    tr = objects.track(LOOP)
    objects.box((0.4, 0.4, 0.4), (0.6, 0.6, 0.6), track=tr)
    for kw in (dict(trans_vel=(0.1, 0, 0)), dict(omega=(0, 1, 0)), dict(dsdt=0.1)):
        with pytest.raises(ValueError):
            objects.box((0.4, 0.4, 0.4), (0.6, 0.6, 0.6), track=tr, **kw)
    with pytest.raises(ValueError):
        objects.sphere((0.5, 0.5, 0.5), 0.1, track=LOOP)


def test_kernel_entry_rejects_before_any_launch():
    """block_count 0: an entry that let a bad argument through would return 0 without a launch"""
    import claymore_b200 as cb
    L = cb.lib()
    cfg = Config(domain_bits=6)
    objs = (_capi.CollisionObject * 1)(objects.box((0.1, 0.1, 0.1), (0.9, 0.2, 0.9)))
    moving = (_capi.CollisionObject * 1)(objects.box((0.1, 0.1, 0.1), (0.9, 0.2, 0.9), trans_vel=(0, 0.1, 0)))
    rec = C.c_void_p(16)   # never read: nothing is launched

    def call(o, spans, records=rec):
        sp = (_capi.TrackSpan * 1)(*spans) if spans is not None else None
        return L.cb200_update_grid_velocity_query_max_tracks(C.byref(cfg), 0, None, _capi.Partition(), 1e-4, None, o, 1, None, 0, records, sp, 0.0, None, None, None)
    assert call(objs, [_capi.TrackSpan(0, 3, 0)]) == 0
    assert call(objs, None) != 0
    assert call(moving, [_capi.TrackSpan(0, 3, 0)]) != 0
    assert call(objs, [_capi.TrackSpan(0, 3, 8)]) != 0
    assert call(objs, [_capi.TrackSpan(-1, 3, 0)]) != 0
    assert call(objs, [_capi.TrackSpan(0, -1, 0)]) != 0
    assert call(objs, [_capi.TrackSpan(0, _capi.MAX_TRACK_KEYS + 1, 0)]) != 0
    assert call(objs, [_capi.TrackSpan(0, 1, _capi.TRACK_PERIODIC)]) != 0
    assert call(objs, [_capi.TrackSpan(0, 3, 0)], None) != 0
    assert call(moving, [_capi.TrackSpan(0, 0, 0)]) == 0      # untracked: the reference motion model as before


def _scene_entry(track):
    return {"boundaries": [{"shape": "box", "offset": [0.4, 0.4, 0.4], "span": [0.2, 0.1, 0.2], "track": track}]}


SCENE_REJECTED = {
    "not_a_dict": [1, 2],
    "unknown_key": {"keys": [{"t": 0}], "speed": 1},
    "no_keys": {"keys": []},
    "key_without_t": {"keys": [{"position": [0.5, 0.5, 0.5]}]},
    "unknown_key_key": {"keys": [{"t": 0, "angle": 1}]},
    "not_increasing": {"keys": [{"t": 0.1}, {"t": 0.1}]},
    "periodic_mismatch": {"keys": [{"t": 0}, {"t": 0.1, "position": [0.4, 0.4, 0.4]}], "periodic": True},
    "rotation_shape": {"keys": [{"t": 0}, {"t": 0.1, "rotation": [0, 1.0]}]},
    "bad_interp": {"keys": [{"t": 0}], "interp": "cubic"},
    "non_finite": {"keys": [{"t": 0, "position": [0.5, float("nan"), 0.5]}]},
}


@pytest.mark.parametrize("name", list(SCENE_REJECTED))
def test_scene_rejects_bad_track(name):
    with pytest.raises(ValueError):
        scene.boundaries(_scene_entry(SCENE_REJECTED[name]))


def test_scene_track_pivot_and_velocity_conflict():
    o = scene.boundaries(_scene_entry({"keys": [{"t": 0.0}, {"t": 0.2, "position": [0.5, 0.3, 0.5], "rotation": [0, 0.5, 0]}], "interp": "smooth"}))[0]
    assert list(o.trans) == pytest.approx([0.5, 0.45, 0.5]) and o.track.n == 2 and o.track.flags == _capi.TRACK_SMOOTH
    assert list(o.track.keys[0].pos) == pytest.approx([0.5, 0.45, 0.5])
    assert list(o.track.keys[1].rot) == pytest.approx([np.cos(0.25), 0, np.sin(0.25), 0])
    plane = scene.boundaries({"boundaries": [{"shape": "plane", "offset": [0.5, 0.2, 0.5], "track": {"keys": [{"t": 0}]}}]})[0]
    assert list(plane.trans) == pytest.approx([0.5, 0.2, 0.5])
    bad = _scene_entry({"keys": [{"t": 0}]})
    bad["boundaries"][0]["velocity"] = [0, 1, 0]
    with pytest.raises(ValueError):
        scene.boundaries(bad)
    with pytest.raises(ValueError):   # sinks take no track
        scene.sinks({"sinks": [{"shape": "box", "offset": [0.4, 0.4, 0.4], "span": [0.1, 0.1, 0.1], "track": {"keys": [{"t": 0}]}}]})


def _rot(e, R0=np.eye(3)):
    return RT.quat_mat(e["q"]) @ R0


def _check_derivatives(rec, flags, t, label, h=1e-4):
    """c' and omega of the float64 evaluation at t against central differences of c(t) and R(t) (R' = [omega]x R); h well above the
    float32 u's resolution"""
    e = RT.evaluate(rec, flags, t)
    lo, hi = RT.evaluate(rec, flags, t - h), RT.evaluate(rec, flags, t + h)
    if lo["seg"] != e["seg"] or hi["seg"] != e["seg"]:
        return False                                    # float32 t +- h left the segment: not a point inside one
    dt = hi["tw"] - lo["tw"]
    dc = (hi["c"] - lo["c"]) / dt
    assert np.abs(dc - e["v"]).max() <= 1e-3 * (1 + np.abs(e["v"]).max()), f"{label}: c' {e['v']} vs finite difference {dc}"
    dR = (_rot(hi) - _rot(lo)) / dt
    W = dR @ _rot(e).T
    w = np.array([W[2, 1], W[0, 2], W[1, 0]])
    assert np.abs(w - e["w"]).max() <= 1e-3 * (1 + np.abs(e["w"]).max()), f"{label}: omega {e['w']} vs finite difference {w}"
    return True


@pytest.mark.parametrize("flags", [0, 1, 2, 3])
def test_evaluation_derivatives(flags):
    keys = KEYS
    rec = RT.prepare(keys, flags)
    inside = 0
    for t in np.linspace(0.013, 0.487, 23):
        inside += _check_derivatives(rec, flags, float(t), f"flags {flags} t {t}")
    assert inside >= 20
    # the keys' poses and the holds
    for k, (tk, p, q) in enumerate(keys[:-1]):
        e = RT.evaluate(rec, flags, tk)
        assert e["seg"] == k and e["u"] == 0.0 and np.allclose(e["c"], p)
        assert np.abs(np.abs(e["q"] @ rec[k, 4:8]) - 1) < 1e-6
    before = RT.evaluate(rec, flags, -0.3)
    assert before["seg"] == -1 and np.allclose(before["c"], keys[0][1]) and not before["v"].any() and not before["w"].any()
    late = 1.3 if flags & _capi.TRACK_PERIODIC else 0.5
    after = RT.evaluate(rec, flags, late)
    if flags & _capi.TRACK_PERIODIC:
        # 1.3 = 0.3 + two periods: the same pose and velocity as at 0.3 (float32 wrap), derivatives inside the wrapped segment
        ref = RT.evaluate(rec, flags, after["tw"])
        assert abs(after["tw"] - 0.3) < 1e-6 and np.allclose(after["c"], ref["c"]) and np.allclose(after["v"], ref["v"])
        assert _check_derivatives(rec, flags, 1.3, "after the wrap")
    else:
        assert after["seg"] == -1 and np.allclose(after["c"], keys[-1][1]) and not after["v"].any()


def test_smooth_is_c1_at_keys_and_one_key_holds():
    rec = RT.prepare(KEYS, 1)
    for k in range(1, len(KEYS) - 1):
        t = float(np.float32(KEYS[k][0]))
        a, b = RT.evaluate(rec, 1, float(np.nextafter(np.float32(t), np.float32(0)))), RT.evaluate(rec, 1, t)
        assert np.abs(a["v"] - b["v"]).max() < 1e-3 * (1 + np.abs(b["v"]).max()), f"key {k}: c' jumps {a['v']} -> {b['v']}"
    one = RT.prepare([(0.0, (0.3, 0.4, 0.5), (1, 0, 0, 0))], 0)
    e = RT.evaluate(one, 0, 0.7)
    assert np.array_equal(e["c"], np.float32([0.3, 0.4, 0.5])) and np.array_equal(e["q"], [1, 0, 0, 0])


def test_one_key_rest_track_frame_is_the_static_frame():
    """A one-key track with c = trans and q = 1 places the object as the untracked static object (ref64.collider_frame)."""
    o = objects.box((0.4, 0.4, 0.4), (0.6, 0.5, 0.6), trans=(0.5, 0.45, 0.5), rot=RT.quat_mat(_q((1, 2, 3), 0.4)),
                    track=objects.track([(0.0, (0.5, 0.45, 0.5), (1, 0, 0, 0))]))
    p = ref64.object_params(o)
    f, g = RT.frame(p, 0.37), ref64.collider_frame(p, 0.37)
    assert np.allclose(f["rot"][0], g["rot"][0], atol=1e-15) and np.array_equal(f["b"][0], g["b"][0])
