"""Writes tests/golden/ref_sdf_*.npz with the reference's own level-set sampler (oracle/_ref/libclaymore_ref_sdf.so, built by
oracle/build_ref_sdf.sh): SampleGenerator::LoadSDF's parse and GenerateUniformSamples' output for small synthetic level sets.

Each file holds the SDFGen text (`text`, uint8), the reference's parse (`dims`, `mins`, `h`, `phi`), V (GenerateUniformSamples with
one sample per cell returns the valid-cell count), gmpm's sampleNum for MODEL_PPC = 8 on a 256^3 grid (read_sdf,
ParticleIO.hpp:79-84: samplesPerCell = 8 min(n) / 256), and the index-space samples of srand(seed) for `seeds` at `spc` samples
per cell.  When the reference checkout has Data/MpmParticles/two_dragons.sdf, ref_sdf_two_dragons.npz gets its header, V, gmpm's
sampleNum and a histogram of the reference's samples over 4^3-cell bins (not the 29 MB file).

    python tests/golden/make_ref_sdf_golden.py
"""
import ctypes as C
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(HERE))
import sdf_ref as R  # noqa: E402

SHIM = os.path.join(ROOT, "oracle", "_ref", "libclaymore_ref_sdf.so")
REFERENCE = os.environ.get("CLAYMORE_REFERENCE", "/root/reference")
SEEDS = (0, 1, 7)

CASES = {
    "sphere": (R.sphere((13, 14, 15), 0.5, (3.0, 3.2, 3.5), 2.6), 4.0),
    "torus": (R.torus((20, 12, 20), 0.25, (2.4, 1.4, 2.4), 1.5, 0.6), 2.0),
    "dragonish": (R.dragonish(), 1.0),
    "plate": (R.plate((10, 10, 8), 0.5, 3), 3.0),
}


def shim():
    L = C.CDLL(SHIM)
    L.ref_sdf_load.argtypes = [C.c_char_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong]
    L.ref_sdf_uniform.argtypes = [C.c_char_p, C.c_uint, C.c_float, C.c_void_p, C.c_longlong]
    L.ref_sdf_uniform.restype = C.c_longlong
    return L


def load(L, path, with_phi=True):
    dims, mins, h = np.zeros(3, np.int32), np.zeros(3, np.float32), np.zeros(1, np.float32)
    L.ref_sdf_load(path.encode(), dims.ctypes.data, mins.ctypes.data, h.ctypes.data, None, 0)
    phi = None
    if with_phi:
        phi = np.zeros(int(np.prod(dims.astype(np.int64))), np.float32)
        L.ref_sdf_load(path.encode(), dims.ctypes.data, mins.ctypes.data, h.ctypes.data, phi.ctypes.data, phi.size)
    return dims, mins, float(h[0]), phi


def uniform(L, path, seed, spc, cap):
    out = np.zeros((cap, 3), np.float32)
    n = L.ref_sdf_uniform(path.encode(), seed, spc, out.ctypes.data, cap)
    return n, out[:n]


def gmpm_sample_num(V, dims):
    spc = np.float32(8.0) * np.float32(int(dims.min())) / np.float32(256)   # read_sdf's float arithmetic
    return int(np.float32(V) * spc)


def main():
    L = shim()
    with tempfile.TemporaryDirectory() as tmp:
        for name, ((n, h, phi), spc) in CASES.items():
            text = R.text(n, h, phi, origin=(-0.5, 0.25, 1.0))
            path = os.path.join(tmp, name + ".sdf")
            with open(path, "wb") as f:
                f.write(text)
            dims, mins, hh, rphi = load(L, path)
            V, _ = uniform(L, path, 0, 1.0, int(np.prod(dims)))
            samples = {}
            for s in SEEDS:
                num, pts = uniform(L, path, s, spc, int(V * spc) + 1)
                samples[f"samples_{s}"] = pts
            np.savez_compressed(os.path.join(HERE, f"ref_sdf_{name}.npz"), text=np.frombuffer(text, np.uint8), dims=dims, mins=mins,
                                h=np.float32(hh), phi=rphi, V=np.int64(V), gmpm_sample_num=np.int64(gmpm_sample_num(V, dims)),
                                spc=np.float32(spc), seeds=np.array(SEEDS), **samples)
            print(name, dims, "V", V, "samples", [len(v) for v in samples.values()])
    dragons = os.path.join(REFERENCE, "Data", "MpmParticles", "two_dragons.sdf")
    if os.path.exists(dragons):
        dims, mins, hh, _ = load(L, dragons, with_phi=False)
        V, _ = uniform(L, dragons, 0, 1.0, 0)
        num, pts = uniform(L, dragons, 0, np.float32(8.0) * np.float32(int(dims.min())) / np.float32(256), gmpm_sample_num(V, dims) + 1)
        bins = [np.arange(0, d + 4, 4) for d in dims - 1]
        hist, _ = np.histogramdd(pts.astype(np.float64), bins=bins)
        np.savez_compressed(os.path.join(HERE, "ref_sdf_two_dragons.npz"), dims=dims, mins=mins, h=np.float32(hh), V=np.int64(V),
                            gmpm_sample_num=np.int64(num), hist=hist.astype(np.int32))
        print("two_dragons", dims, "V", V, "sampleNum", num)
    else:
        print(f"{dragons} not found: no ref_sdf_two_dragons.npz")


if __name__ == "__main__":
    main()
