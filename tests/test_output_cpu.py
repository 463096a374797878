"""CPU tests of the per-frame .bgeo format: the library's host header / trailer (cb200_bgeo_header / cb200_bgeo_trailer) around a
big-endian body built with numpy (the records the device gather writes) against files the reference's own writer produced
(tests/golden/ref_bgeo_*.bgeo, made by tests/golden/make_ref_bgeo_golden.py) and, where oracle/_ref is built, against fresh output of
mn::write_partio / partio and partio's reader; and claymore_b200.bgeo.read with its rejections."""
import ctypes as C
import os
import struct

import numpy as np
import pytest

from claymore_b200 import bgeo
from claymore_b200._capi import OUTPUT_J, OUTPUT_V, lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
SHIM = os.path.join(ROOT, "oracle", "_ref", "libclaymore_ref_partio.so")
CASES = {"pos": (False, False), "v": (True, False), "J": (False, True), "vJ": (True, True), "empty": (True, True), "one": (False, False)}


def header(n, attrs):
    buf = (C.c_ubyte * 256)()
    size = C.c_size_t(0)
    rc = lib().cb200_bgeo_header(n, attrs, buf, 256, C.byref(size))
    assert rc == 0, rc
    return bytes(buf[: size.value])


def trailer():
    buf = (C.c_ubyte * 8)()
    size = C.c_size_t(0)
    assert lib().cb200_bgeo_trailer(buf, 8, C.byref(size)) == 0
    return bytes(buf[: size.value])


def body(pts, with_v, with_j):
    """the device's records: x y z 1.0 [v] [J], big-endian words (bits moved as integers)"""
    cols = [pts[:, :3], np.ones((len(pts), 1), np.float32)]
    if with_v:
        cols.append(pts[:, 3:6])
    if with_j:
        cols.append(pts[:, 6:7])
    rec = np.concatenate([c.view(np.uint32) for c in cols], axis=1)
    return rec.astype(">u4").tobytes()


def library_file(pts, with_v, with_j):
    attrs = (OUTPUT_V if with_v else 0) | (OUTPUT_J if with_j else 0)
    return header(len(pts), attrs) + body(pts, with_v, with_j) + trailer()


def golden_points():
    return dict(np.load(os.path.join(GOLDEN, "ref_bgeo_points.npz")))


@pytest.mark.parametrize("name", sorted(CASES))
def test_library_file_equals_reference_golden(name):
    pts = golden_points()[name]
    want = open(os.path.join(GOLDEN, f"ref_bgeo_{name}.bgeo"), "rb").read()
    assert library_file(pts, *CASES[name]) == want


@pytest.mark.parametrize("name", sorted(CASES))
def test_reader_round_trips_golden_bits(name):
    pts = golden_points()[name]
    with_v, with_j = CASES[name]
    d = bgeo.read(os.path.join(GOLDEN, f"ref_bgeo_{name}.bgeo"))
    assert set(d) == {"position"} | ({"v"} if with_v else set()) | ({"J"} if with_j else set())
    assert d["position"].shape == (len(pts), 3) and d["position"].dtype == np.float32
    assert d["position"].view(np.uint32).tobytes() == np.ascontiguousarray(pts[:, :3]).view(np.uint32).tobytes()
    if with_v:
        assert d["v"].shape == (len(pts), 3) and d["v"].view(np.uint32).tobytes() == np.ascontiguousarray(pts[:, 3:6]).view(np.uint32).tobytes()
    if with_j:
        assert d["J"].shape == (len(pts),) and d["J"].view(np.uint32).tobytes() == np.ascontiguousarray(pts[:, 6]).view(np.uint32).tobytes()


def test_header_rejects_out_of_range():
    buf = (C.c_ubyte * 256)()
    size = C.c_size_t(0)
    L = lib()
    assert L.cb200_bgeo_header(2 ** 31, 0, buf, 256, C.byref(size)) != 0      # the point count is a 32-bit field
    assert L.cb200_bgeo_header(-1, 0, buf, 256, C.byref(size)) != 0
    assert L.cb200_bgeo_header(5, 4, buf, 256, C.byref(size)) != 0           # unknown attribute bit
    assert L.cb200_bgeo_header(5, 3, buf, 10, C.byref(size)) != 0            # capacity below the size
    assert L.cb200_bgeo_header(2 ** 31 - 1, 3, buf, 256, C.byref(size)) == 0
    assert struct.unpack(">i", bytes(buf[9:13]))[0] == 2 ** 31 - 1


def _shim():
    if not os.path.exists(SHIM):
        pytest.skip("oracle/_ref/libclaymore_ref_partio.so not built (oracle/build_ref_partio.sh)")
    import sys
    sys.path.insert(0, GOLDEN)
    import make_ref_bgeo_golden as mk
    return mk, mk.load_shim()


def partio_read(shim, path):
    n, attrs = C.c_longlong(0), C.c_int(0)
    assert shim.ref_read_partio(path.encode(), C.byref(n), C.byref(attrs), None, None, None) == 0
    pos, v, J = (np.zeros((n.value, 3), np.float32), np.zeros((n.value, 3), np.float32), np.zeros(n.value, np.float32))
    assert shim.ref_read_partio(path.encode(), C.byref(n), C.byref(attrs), pos.ctypes.data_as(C.c_void_p), v.ctypes.data_as(C.c_void_p), J.ctypes.data_as(C.c_void_p)) == 0
    return pos, (v if attrs.value & 1 else None), (J if attrs.value & 2 else None)


@pytest.mark.parametrize("n", [0, 1, 2, 33, 1000])
@pytest.mark.parametrize("name", ["pos", "v", "J", "vJ"])
def test_library_file_equals_fresh_reference_output(tmp_path, name, n):
    mk, shim = _shim()
    with_v, with_j = CASES[name]
    pts = mk.special_points(n, 7 * n + len(name))
    path = str(tmp_path / "ref.bgeo")
    mk.write(shim, path, pts, with_v, with_j)
    mine = library_file(pts, with_v, with_j)
    assert mine == open(path, "rb").read()
    # partio reads the library's file back with every bit (-0.0, NaN payloads, denormals)
    lib_path = str(tmp_path / "lib.bgeo")
    open(lib_path, "wb").write(mine)
    pos, v, J = partio_read(shim, lib_path)
    assert pos.view(np.uint32).tobytes() == np.ascontiguousarray(pts[:, :3]).view(np.uint32).tobytes()
    assert (v is not None) == with_v and (J is not None) == with_j
    if with_v:
        assert v.view(np.uint32).tobytes() == np.ascontiguousarray(pts[:, 3:6]).view(np.uint32).tobytes()
    if with_j:
        assert J.view(np.uint32).tobytes() == np.ascontiguousarray(pts[:, 6]).view(np.uint32).tobytes()


def _malformed():
    good = open(os.path.join(GOLDEN, "ref_bgeo_vJ.bgeo"), "rb").read()
    pos = open(os.path.join(GOLDEN, "ref_bgeo_pos.bgeo"), "rb").read()

    def field(data, i, value):   # i-th int32 after "BgeoV"
        return data[: 5 + 4 * i] + struct.pack(">i", value) + data[9 + 4 * i:]
    # the J attribute (the last definition of the vJ file) given type 1 (int) / 4 (indexed string)
    j_type = good.index(b"\x00\x01J") + 5
    return {
        "bad magic": b"Bgeq" + good[4:],
        "new-format magic": b"\x7fNSJ" + good[4:],
        "version 4": field(good, 0, 4),
        "header only partly there": good[:30],
        "truncated in the attribute definitions": good[:50],
        "truncated in the records": good[:-10],
        "missing trailer": good[:-2],
        "trailing bytes": good + b"\x00",
        "primitives": field(pos, 2, 1),
        "point groups": field(pos, 3, 1),
        "primitive groups": field(pos, 4, 1),
        "int attribute": good[:j_type] + struct.pack(">i", 1) + good[j_type + 4:],
        "indexed string attribute": good[:j_type] + struct.pack(">i", 4) + good[j_type + 4:],
    }


@pytest.mark.parametrize("case", sorted(_malformed()))
def test_reader_rejects_malformed(tmp_path, case):
    p = tmp_path / "bad.bgeo"
    p.write_bytes(_malformed()[case])
    with pytest.raises(ValueError):
        bgeo.read(str(p))
