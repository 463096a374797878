"""Particle models from SDFGen `.sdf` level sets (the reference's read_sdf, Library/MnSystem/IO/ParticleIO.hpp:65-97).

    ls = sdf.read("dragon.sdf")                                  # the library's parser (strtof: LoadSDF's values bit for bit)
    sdf.write(ls, "copy.sdf")                                    # SDFGen text, 9 significant digits: read() returns ls bit for bit
    pos = sdf.sample(ls, cfg, offset, span, ppc=8)               # host positions, e.g. for samplers.split_slabs
    sim.init_model_sdf(material, ls, offset, span, v0)           # sampled straight into the model's device array

Placement: one scale for all axes, c = min_d span_d / ((n_d - 1) h) * h; node q lands at offset + q c, and the node box
[offset, offset + (n - 1) c] must lie inside the domain [0, 1]^3.  Modes (include/claymore_b200.h, DESIGN §2.7): "random" (the
reference's sampler with its quirks S1-S4 fixed; ppc particles per simulation cell on average) and "lattice" (ppc = k^3 points per
simulation cell, samplers.uniform_box's pattern for k = 2, masked by the level set).
"""
import ctypes as C

import numpy as np

from ._capi import SDF_LATTICE, SDF_RANDOM, CB200Error, SdfHeader, SdfSampling, check, lib

MODES = {"random": SDF_RANDOM, "lattice": SDF_LATTICE}


class LevelSet:
    """A parsed level set: n = (ni, nj, nk) nodes, spacing h, SDFGen origin `min` (metadata), phi float32 with i fastest."""

    def __init__(self, header, phi):
        self.header = header
        self.phi = phi

    @property
    def n(self):
        return (self.header.ni, self.header.nj, self.header.nk)

    @property
    def h(self):
        return float(self.header.h)

    @property
    def grid(self):
        """phi as an array indexed [k, j, i]."""
        return self.phi.reshape(self.n[::-1])


def parse(text):
    """Parses SDFGen text (bytes or str).  Raises ValueError for anything cb200_sdf_parse rejects."""
    if isinstance(text, str):
        text = text.encode()
    hdr = SdfHeader()
    if lib().cb200_sdf_parse(text, len(text), C.byref(hdr), None, 0) != 0:
        raise ValueError("not a valid .sdf level set (dimensions >= 2 with fewer than 2^31 nodes, h finite and > 0, "
                         "exactly ni nj nk finite values)")
    phi = np.empty(hdr.ni * hdr.nj * hdr.nk, np.float32)
    check(lib().cb200_sdf_parse(text, len(text), C.byref(hdr), phi.ctypes.data_as(C.c_void_p), phi.size), "sdf_parse")
    return LevelSet(hdr, phi)


def read(path):
    with open(path, "rb") as f:
        return parse(f.read())


def write(ls, path):
    """Writes `ls` as SDFGen text with 9 significant digits, so that read(path) returns ls bit for bit."""
    n = ls.n
    with open(path, "w") as f:
        f.write(f"{n[0]} {n[1]} {n[2]}\n{' '.join('%.9g' % float(v) for v in ls.header.min)}\n{'%.9g' % ls.h}\n")
        np.savetxt(f, np.asarray(ls.phi, dtype=np.float32).reshape(-1, 1), fmt="%.9g")


def _vec3(v):
    a = np.broadcast_to(np.asarray(v, dtype=np.float64), (3,))
    return [float(x) for x in a]


def node_box(ls, offset, span):
    """(c, lo, hi): the world size of one level-set cell and the node box, computed as the library does (double)."""
    offset, span = _vec3(offset), _vec3(span)
    h = float(np.float32(ls.h))
    s = min(span[d] / (float(ls.n[d] - 1) * h) for d in range(3))
    c = s * h
    return c, offset, [offset[d] + float(ls.n[d] - 1) * c for d in range(3)]


def check_box(ls, offset, span, what="level set"):
    """Raises ValueError unless span > 0 and the node box lies inside [0, 1]^3; the message names `what` and the box."""
    if min(_vec3(span)) <= 0:
        raise ValueError(f"{what}: span {_vec3(span)} must be positive")
    c, lo, hi = node_box(ls, offset, span)
    if not all(lo[d] >= 0.0 and hi[d] <= 1.0 for d in range(3)):
        raise ValueError(f"{what}: node box [{', '.join(f'{v:.6g}' for v in lo)}] - [{', '.join(f'{v:.6g}' for v in hi)}] "
                         f"(cell {c:.6g}) does not lie inside the domain [0, 1]^3")
    return c, lo, hi


def sampling(offset, span, ppc=8, mode="random", seed=0):
    if mode not in MODES:
        raise ValueError(f"unknown sdf sampler {mode!r} (known: {', '.join(MODES)})")
    smp = SdfSampling()
    smp.mode, smp.ppc, smp.seed = MODES[mode], int(ppc), int(seed) & 0xFFFFFFFFFFFFFFFF
    smp.offset[:], smp.span[:] = _vec3(offset), _vec3(span)
    return smp


def sample(ls, cfg, offset, span, ppc=8, mode="random", seed=0, stream=None):
    """Samples the level set on the current device; returns float32 positions (count, 3) in candidate order."""
    check_box(ls, offset, span)
    smp = sampling(offset, span, ppc, mode, seed)
    phi = np.ascontiguousarray(ls.phi, dtype=np.float32)
    n = C.c_longlong(0)
    args = (C.byref(cfg), C.byref(ls.header), phi.ctypes.data_as(C.c_void_p), C.byref(smp))
    st = C.c_void_p(stream) if stream else None
    check(lib().cb200_sample_sdf(*args, None, 0, C.byref(n), st), "sample_sdf")
    out = np.empty((n.value, 3), np.float32)
    if n.value:
        check(lib().cb200_sample_sdf(*args, out.ctypes.data_as(C.c_void_p), n.value, C.byref(n), st), "sample_sdf")
    return out


__all__ = ["LevelSet", "MODES", "parse", "read", "write", "node_box", "check_box", "sampling", "sample", "CB200Error"]
