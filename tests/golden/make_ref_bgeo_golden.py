"""Writes the .bgeo golden files of tests/test_output_cpu.py with the reference's own writer (oracle/_ref/libclaymore_ref_partio.so,
built by oracle/build_ref_partio.sh): mn::write_partio for positions only, partio's addAttribute("v", VECTOR, 3) / ("J", FLOAT, 1)
for the others.  The points (seeded, with -0.0, NaN payloads and denormals among them) go to ref_bgeo_points.npz.

    python tests/golden/make_ref_bgeo_golden.py
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
SHIM = os.path.join(ROOT, "oracle", "_ref", "libclaymore_ref_partio.so")

# name -> (points, with v, with J)
CASES = {"pos": (7, False, False), "v": (7, True, False), "J": (7, False, True), "vJ": (7, True, True), "empty": (0, True, True), "one": (1, False, False)}


def special_points(n, seed):
    """float32 [n, 7] (x y z vx vy vz J) from a seed, with the bit patterns a writer must not change put in the first rows"""
    rng = np.random.default_rng(seed)
    a = rng.uniform(-2.0, 2.0, (n, 7)).astype(np.float32)
    bits = a.view(np.uint32)
    special = [0x80000000, 0x7FC12345, 0xFFA00001, 0x00000001, 0x807FFFFF, 0x7F800000, 0x3F800000]  # -0, NaNs, denormals, inf, 1
    for i in range(min(n, 3)):
        bits[i] = np.roll(np.array(special, np.uint32), i)[: a.shape[1]]
    return a


def write(shim, path, pts, with_v, with_j):
    pos = np.ascontiguousarray(pts[:, :3])
    v = np.ascontiguousarray(pts[:, 3:6]) if with_v else None
    J = np.ascontiguousarray(pts[:, 6]) if with_j else None
    p = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    if not with_v and not with_j:
        rc = shim.ref_write_partio(path.encode(), p(pos), C.c_longlong(len(pts)))
    else:
        rc = shim.ref_write_partio_attributes(path.encode(), p(pos), p(v), p(J), C.c_longlong(len(pts)))
    assert rc == 0


def load_shim():
    lib = C.CDLL(SHIM)
    lib.ref_write_partio.argtypes = [C.c_char_p, C.c_void_p, C.c_longlong]
    lib.ref_write_partio_attributes.argtypes = [C.c_char_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong]
    lib.ref_read_partio.argtypes = [C.c_char_p, C.POINTER(C.c_longlong), C.POINTER(C.c_int), C.c_void_p, C.c_void_p, C.c_void_p]
    return lib


def main():
    shim = load_shim()
    points = {}
    for k, (name, (n, with_v, with_j)) in enumerate(sorted(CASES.items())):
        pts = special_points(n, 1000 + k)
        points[name] = pts
        write(shim, os.path.join(HERE, f"ref_bgeo_{name}.bgeo"), pts, with_v, with_j)
    np.savez(os.path.join(HERE, "ref_bgeo_points.npz"), **points)
    print("wrote", ", ".join(f"ref_bgeo_{n}.bgeo" for n in sorted(CASES)), "and ref_bgeo_points.npz")


if __name__ == "__main__":
    main()
