"""Reading checkpoints written by GmpmSimulator.save_checkpoint / checkpoint_end (layout: include/claymore_b200.h).

The blob is parsed and validated by the library's one parser, cb200_checkpoint_inspect (host only, no device needed); this
module only maps the sections it reports.  A file is memory-mapped, so reading a multi-GB checkpoint touches only the pages
that are used.
"""
import ctypes as C

import numpy as np

from ._capi import CHANNELS, CheckpointInfo, check, lib

PARAMS = ("rho", "volume", "mass", "bulk", "gamma", "viscosity", "lambda_", "mu", "cohesion", "beta", "yield_surface",
          "volume_correction", "bm", "xi", "msqr", "hardening_on")


def _map(path_or_buffer):
    if isinstance(path_or_buffer, np.ndarray):
        return np.ascontiguousarray(path_or_buffer).view(np.uint8).reshape(-1)
    if isinstance(path_or_buffer, (bytes, bytearray, memoryview)):
        return np.frombuffer(path_or_buffer, np.uint8)
    return np.memmap(path_or_buffer, dtype=np.uint8, mode="r")


def inspect(path_or_buffer):
    """(CheckpointInfo, uint8 view of the blob); raises CB200Error when the library rejects the blob."""
    blob = _map(path_or_buffer)
    inf = CheckpointInfo()
    check(lib().cb200_checkpoint_inspect(C.c_void_p(blob.ctypes.data if blob.size else 0), blob.size, C.byref(inf)), "checkpoint_inspect")
    return inf, blob


def _as_dict(inf):
    d = {k: getattr(inf, k) for k, _ in CheckpointInfo._fields_ if k not in ("cfg", "models")}
    d["cfg"] = {k: getattr(inf.cfg, k) for k, _ in inf.cfg._fields_}
    d["models"] = []
    for m in inf.models[: inf.n_models]:
        p = {k: getattr(m.params, k) for k in PARAMS}
        p["lambda"] = p.pop("lambda_")
        d["models"].append(dict(material=m.material, channels=m.channels, count=m.count, offset=m.offset, bytes=m.bytes, params=p))
    return d


def info(path_or_buffer):
    """Header and table of contents of a checkpoint as a dict: config, clock, block counts, and per model its material,
    parameters, particle count and section."""
    return _as_dict(inspect(path_or_buffer)[0])


def read(path_or_buffer):
    """info() plus numpy views of the data: "states" (per model float32[count, channels], the layout of particle_state),
    "keys" (int32[nbc, 3]) and "grid" (float32[nbc, 4, 64]: mass, momentum x, y, z of every cell)."""
    inf, blob = inspect(path_or_buffer)
    out = _as_dict(inf)
    out["states"] = [blob[m.offset: m.offset + m.bytes].view("<f4").reshape(m.count, CHANNELS[m.material]) for m in inf.models[: inf.n_models]]
    nbc = inf.neighbor_block_count
    out["keys"] = blob[inf.keys_offset: inf.keys_offset + inf.keys_bytes].view("<i4").reshape(nbc, 3)
    out["grid"] = blob[inf.grid_offset: inf.grid_offset + inf.grid_bytes].view("<f4").reshape(nbc, 4, 64)
    return out
