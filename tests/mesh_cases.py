"""Meshes and lattices for the mesh level-set tests (claymore_b200.mesh), the float32 header of SDFGen's main, and the binding of
SDFGen itself (oracle/_ref/libclaymore_ref_sdfgen.so, built by oracle/build_ref_sdfgen.sh) when it has been built."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden")
TORUS_NPZ = os.path.join(GOLDEN, "torus-tri-10k.npz")   # the reference's Data/TriMesh/torus-tri-10k.obj as float32 / int32 arrays
SHIM = os.path.join(ROOT, "oracle", "_ref", "libclaymore_ref_sdfgen.so")

CUBE_F = [[0, 2, 1], [0, 3, 2], [4, 5, 6], [4, 6, 7], [0, 1, 5], [0, 5, 4], [1, 2, 6], [1, 6, 5], [2, 3, 7], [2, 7, 6], [3, 0, 4], [3, 4, 7]]
CUBE_V = [[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0], [0, 0, 1], [1, 0, 1], [1, 1, 1], [0, 1, 1]]


def cube(lo=(0, 0, 0), size=1.0):
    return np.asarray(CUBE_V, np.float32) * np.float32(size) + np.asarray(lo, np.float32), np.asarray(CUBE_F, np.int32)


def plain_obj(v, t):
    """SDFGen-readable OBJ text: `v` with 9 significant digits (float32 round trip), `f` 1-based."""
    lines = ["v %.9g %.9g %.9g" % tuple(float(c) for c in p) for p in v] + ["f %d %d %d" % tuple(int(i) + 1 for i in f) for f in t]
    return "\n".join(lines) + "\n"


def torus():
    """vertices / triangles of the 10 k-triangle torus"""
    g = np.load(TORUS_NPZ)
    return g["vertices"], g["triangles"]


def write_torus_obj(path):
    """the torus as a plain OBJ file at `path` (every float32 round-trips through its 9 digits)"""
    with open(path, "w") as fh:
        fh.write(plain_obj(*torus()))
    return str(path)


def golden(path):
    """a recorded golden as a dict, the torus cases' mesh filled in from TORUS_NPZ"""
    g = dict(np.load(path))
    if "vertices" not in g:
        g["vertices"], g["triangles"] = torus()
    return g


def cases():
    """{name: (vertices, triangles, h, padding, exact_band)} of the recorded goldens."""
    tv, tt = torus()
    out = {
        "torus_h07_p1_b1": (tv, tt, 0.07, 1, 1),
        "torus_h07_p3_b0": (tv, tt, 0.07, 3, 0),
        "torus_h055_p1_b3": (tv, tt, 0.055, 1, 3),
        "torus_h055_p3_b1": (tv, tt, 0.055, 3, 1),
        "torus_h045_p1_b1": (tv, tt, 0.045, 1, 1),
    }
    v, t = cube()
    out["cube_on_nodes"] = (v, t, 0.125, 1, 1)          # vertices and edges on lattice nodes: the SOS branches, fi on integers
    out["open_box"] = (v, t[2:], 0.1, 2, 1)             # no bottom: parity streaks
    v2, t2 = cube((0.5, 0.25, 0.375), 1.0)
    out["two_bodies"] = (np.vstack([v, v2]), np.vstack([t, t2 + 8]), 0.0625, 1, 2)
    rng = np.random.default_rng(5)
    vd = np.vstack([v, [[0.2, 0.3, 0.4], [0.6, 0.7, 0.8], [0.4, 0.5, 0.6]]]).astype(np.float32)
    out["degenerate"] = (vd, np.vstack([t, [[8, 9, 10], [8, 8, 9], [1, 1, 1]]]).astype(np.int32), 0.07, 1, 1)
    out["single_triangle"] = (np.asarray([[0.1, 0.2, 0.05], [1.3, 0.4, 0.25], [0.5, 1.1, 0.9]], np.float32), np.asarray([[0, 1, 2]], np.int32), 0.05, 2, 1)
    out["floor"] = (np.asarray([[0, 0, 0], [2, 0, 0], [2, 0, 2], [0, 0, 2]], np.float32), np.asarray([[0, 1, 2], [0, 2, 3]], np.int32), 2.0 / 300, 1, 1)
    extra = (rng.random((5, 3)) * 1.6 - 0.3).astype(np.float32)
    out["unreferenced"] = (np.vstack([[[0.5, 0.5, 0.5]], v, extra]).astype(np.float32), t + 1, 0.08, 1, 1)
    return out


def sdfgen_box(v):
    """SDFGen's vertex box (main.cpp:90 with util.h's update_minmax, `if(a<min) min=a; else if(a>max) max=a;`): the first vertex
    never raises the max (quirk M8)."""
    lo = np.full(3, np.finfo(np.float32).max, np.float32)
    hi = -lo
    for p in np.asarray(v, np.float32):
        for d in range(3):
            if p[d] < lo[d]:
                lo[d] = p[d]
            elif p[d] > hi[d]:
                hi[d] = p[d]
    return lo, hi


def header(v, h, padding, box=None):
    """SDFGen's main (main.cpp:63-118) in float32: (n[3], min[3]) over the vertex box `box` (default: the true one)."""
    f = np.float32
    h = f(h)
    pad = f(max(int(padding), 1)) * h
    lo, hi = box if box is not None else (v.min(axis=0), v.max(axis=0))
    lo, hi = lo - pad, hi + pad
    n = ((hi - lo) / h).astype(np.float32)
    return [int(x) for x in n], lo.astype(np.float32)


def shim():
    if not os.path.exists(SHIM):
        return None
    L = C.CDLL(SHIM)
    L.ref_sdfgen_make_level_set3.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_float, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    L.ref_sdfgen_main.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p]
    return L


def ref_level_set(L, v, t, h, padding, band):
    """SDFGen's make_level_set3 on the float32 header: (n, origin, phi)."""
    n, lo = header(v, h, padding)
    v = np.ascontiguousarray(v, np.float32)
    t = np.ascontiguousarray(t, np.int32)
    phi = np.empty(n[0] * n[1] * n[2], np.float32)
    L.ref_sdfgen_make_level_set3(v.ctypes.data, len(v), t.ctypes.data, len(t), np.ascontiguousarray(lo).ctypes.data, h, n[0], n[1], n[2], band,
                                 phi.ctypes.data)
    return n, lo, phi


def ref_main(obj_text, h, padding):
    """SDFGen's whole main on a copy of the text, in a child process (main exits the process on a bad file and prints to stdout):
    (dims, the origin line's tokens, h token, phi as printed with 6 significant digits)."""
    d = tempfile.mkdtemp()
    try:
        p = os.path.join(d, "m.obj")
        with open(p, "w") as fh:
            fh.write(obj_text)
        code = ("import ctypes as C, sys; L = C.CDLL(sys.argv[1]); L.ref_sdfgen_main.argtypes = [C.c_char_p] * 3; "
                "sys.exit(L.ref_sdfgen_main(*[a.encode() for a in sys.argv[2:]]))")
        subprocess.run(["python3", "-c", code, SHIM, p, repr(float(h)), str(padding)], check=True, stdout=subprocess.DEVNULL, cwd=d)
        with open(os.path.join(d, "m.sdf")) as fh:
            tok = fh.read().split()
        dims = [int(x) for x in tok[:3]]
        return dims, tok[3:6], tok[6], np.asarray(tok[7:], np.float64)
    finally:
        shutil.rmtree(d)
