"""Reading the per-frame particle files GmpmSimulator.write_frame / main_loop(output=...) write: point-only BGEO V5, the layout
partio's writeBGEO produces (the library's writer is byte-identical to it).

Only what such files hold is accepted: the magic "Bgeo", 'V', version 5, points with FLOAT (0) or VECTOR (5) attributes, and
no primitives, groups, vertex or detail attributes.  Anything else raises ValueError.
"""
import struct

import numpy as np

_FLOAT, _VECTOR = 0, 5
TRAILER = b"\x00\xff"


def parse(data):
    """{"position": float32 (n, 3), <attribute name>: float32 (n, size) or (n,) for size 1} from the bytes of a file."""
    data = memoryview(data).cast("B")
    if len(data) < 41:
        raise ValueError("not a BGEO file: shorter than its header")
    if bytes(data[:5]) != b"BgeoV":
        raise ValueError("not a BGEO file: bad magic")
    version, points, prims, point_groups, prim_groups, nattr, vertex_attrs, prim_attrs, detail_attrs = struct.unpack(">9i", data[5:41])
    if version != 5:
        raise ValueError(f"BGEO version {version}: only version 5 is read")
    if points < 0:
        raise ValueError("negative point count")
    if prims or prim_attrs:
        raise ValueError("BGEO file with primitives: only point files are read")
    if point_groups or prim_groups:
        raise ValueError("BGEO file with groups: only point files are read")
    if vertex_attrs or detail_attrs:
        raise ValueError("BGEO file with vertex or detail attributes: only point attributes are read")
    off, attrs, words = 41, [], 4
    for _ in range(nattr):
        if off + 2 > len(data):
            raise ValueError("truncated attribute definition")
        (n,) = struct.unpack(">h", data[off:off + 2])
        if n < 0 or off + 2 + n + 6 > len(data):
            raise ValueError("truncated attribute definition")
        name = bytes(data[off + 2:off + 2 + n]).decode("ascii", "replace")
        size, kind = struct.unpack(">Hi", data[off + 2 + n:off + 8 + n])
        if kind not in (_FLOAT, _VECTOR):
            raise ValueError(f"attribute {name!r} has BGEO type {kind}: only float and vector attributes are read")
        off += 8 + n + 4 * size   # + the zero defaults
        if off > len(data):
            raise ValueError("truncated attribute defaults")
        attrs.append((name, words, size))
        words += size
    end = off + 4 * words * points
    if end + len(TRAILER) > len(data):
        raise ValueError("truncated point records")
    if bytes(data[end:end + len(TRAILER)]) != TRAILER or end + len(TRAILER) != len(data):
        raise ValueError("bad trailer: expected 0x00 0xff right after the point records")
    # swapped as integers, so that every bit pattern (NaN payloads included) arrives unchanged
    rec = np.frombuffer(data, ">u4", count=words * points, offset=off).astype("<u4").view(np.float32).reshape(points, words)
    out = {"position": np.ascontiguousarray(rec[:, :3])}
    for name, w, size in attrs:
        a = np.ascontiguousarray(rec[:, w:w + size])
        out[name] = a[:, 0] if size == 1 else a
    return out


def read(path):
    """The arrays of one .bgeo file: "position" (n, 3) and, where the file has them, "v" (n, 3) and "J" (n,), float32."""
    with open(path, "rb") as f:
        return parse(f.read())
