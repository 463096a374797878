"""Writes tests/golden/ref_sdfgen_<case>.npz with SDFGen itself (oracle/_ref/libclaymore_ref_sdfgen.so, built by
oracle/build_ref_sdfgen.sh): for every case of tests/mesh_cases.cases(), the mesh (`vertices`, `triangles`), `h`, `padding`,
`exact_band` (the torus cases name `mesh` = "torus" instead: its arrays are tests/golden/torus-tri-10k.npz), the float32 header of SDFGen's main (`dims`, `origin`) and make_level_set3's `phi` on it.  Each case is also run
through SDFGen's whole main, whose dims and printed origin (6 significant digits) must equal the header over SDFGen's own vertex
box (quirk M8: the first vertex never raises the max), and, where that box is the true one and the band is main's default 1, whose
printed values must equal `phi` so printed.  The torus is the reference's Data/TriMesh/torus-tri-10k.obj; with the reference
checkout present, tests/golden/torus-tri-10k.npz is first rewritten from it (its `v` / `f a b c` lines, parsed with strtof).

    python tests/golden/make_ref_sdfgen_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import mesh_cases as M  # noqa: E402


REFERENCE = os.environ.get("CLAYMORE_REFERENCE", "/root/reference")


def torus_from_reference():
    import ctypes as C
    strtof = C.CDLL(None).strtof
    strtof.restype, strtof.argtypes = C.c_float, [C.c_char_p, C.c_void_p]
    v, t = [], []
    with open(os.path.join(REFERENCE, "Data", "TriMesh", "torus-tri-10k.obj")) as fh:
        for line in fh:
            s = line.split()
            if s and s[0] == "v":
                v.append([strtof(x.encode(), None) for x in s[1:4]])
            elif s and s[0] == "f":
                t.append([int(x) - 1 for x in s[1:4]])
    np.savez_compressed(M.TORUS_NPZ, vertices=np.asarray(v, np.float32), triangles=np.asarray(t, np.int32))


def main():
    L = M.shim()
    if L is None:
        sys.exit(f"{M.SHIM} not built: run oracle/build_ref_sdfgen.sh")
    if os.path.isdir(REFERENCE):
        torus_from_reference()
    tv, _ = M.torus()
    for name, (v, t, h, padding, band) in M.cases().items():
        n, lo, phi = M.ref_level_set(L, v, t, h, padding, band)
        # main's own box differs from the true one where the first vertex is the only one at a maximum (M8, the torus in x)
        box = M.sdfgen_box(v)
        sn, slo = M.header(v, h, padding, box)
        dims, org, htok, printed = M.ref_main(M.plain_obj(v, t), h, padding)
        assert dims == sn, (name, dims, sn)
        assert org == ["%g" % float(x) for x in slo], (name, org, slo)
        if band == 1 and sn == n:   # main runs make_level_set3 with its default band
            assert np.array_equal(printed, np.asarray(["%g" % float(x) for x in phi], np.float64)), name
        mesh = {"mesh": "torus"} if v is tv else {"vertices": v, "triangles": t}
        np.savez_compressed(os.path.join(HERE, f"ref_sdfgen_{name}.npz"), **mesh, h=np.float32(h), padding=padding, exact_band=band,
                            dims=np.asarray(n, np.int32), origin=lo, phi=phi)
        print(f"{name}: {n} nodes, phi in [{phi.min():.4g}, {phi.max():.4g}], {(phi < 0).sum()} negative")


if __name__ == "__main__":
    main()
