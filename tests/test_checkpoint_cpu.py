"""CPU tests of the checkpoint format: the ctypes mirror of cb200_checkpoint_info, the one parser (cb200_checkpoint_inspect, host
only) on blobs written here by a test-local writer that follows the layout documented in include/claymore_b200.h, every rejection
of its validation list, 64-bit offsets past 2^31 bytes, and the scene front-end's resume check."""
import ctypes as C
import json
import os
import struct
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = 1024
TOC = 96
CHANNELS = {0: 4, 1: 12, 2: 13, 3: 13}
PARAM_FMT = "<11fi3fi"   # rho .. yield_surface, volume_correction, bm, xi, msqr, hardening_on


def _align(x):
    return (x + 255) & ~255


def _params(i):
    return (1000.0 + i, 1e-6, 1e-3, 4e4, 7.15, 0.01, 1.25e3 + i, 3.5e3, 0.0, 0.5, 0.81, 1, 3.1e3, 0.8, 3.42, 1)


def make_blob(models=None, nbc=None, cfg=(6, 128, 2, -9.8, 0.5), clock=None, seed=0, layout=None, header_only=False):
    """A checkpoint as the documented layout describes it.  models: [(material, count)]; the data are seeded random values.
    layout(hdr, toc) may edit the header fields before they are packed (corruption tests); header_only returns the header alone."""
    rng = np.random.default_rng(seed)
    models = models if models is not None else [(1, 300), (0, 70)]
    G = 1 << (cfg[0] - 2)
    if nbc is None:
        nbc = 40
    flat = rng.choice(G ** 3, size=nbc, replace=False)
    keys = np.stack([flat // (G * G), (flat // G) % G, flat % G], 1).astype("<i4")
    grid = rng.standard_normal((nbc, 4, 64)).astype("<f4")
    states = [rng.standard_normal((n, CHANNELS[mat])).astype("<f4") for mat, n in models]
    off = HEADER
    toc = []
    for (mat, n), st in zip(models, states):
        toc.append(dict(material=mat, channels=CHANNELS[mat], count=n, offset=off, bytes=st.nbytes))
        off = _align(off + st.nbytes)
    keys_off = off
    grid_off = _align(keys_off + keys.nbytes)
    total = grid_off + grid.nbytes
    c = dict(dt=1e-4, next_dt=9e-5, step_time=0.0123, frame_time=1 / 24, sim_time=0.456789, steps=4567, frames=10, error=0, dt_default=1e-4, fps=24,
             rank=0, world=1, pbc=min(10, nbc), nbc=nbc, ebc=nbc + 25, max_blocks=4000)
    c.update(clock or {})
    hdr = dict(magic=b"CB200CKP", version=1, n_models=len(models), bytes=total, keys_offset=keys_off, keys_bytes=keys.nbytes, grid_offset=grid_off,
               grid_bytes=grid.nbytes, **c)
    if layout is not None:
        layout(hdr, toc)
    buf = bytearray(HEADER if header_only else max(hdr["bytes"], HEADER))
    struct.pack_into("<8sIIQ", buf, 0, hdr["magic"], hdr["version"], hdr["n_models"], hdr["bytes"])
    struct.pack_into("<iiiff", buf, 24, *cfg)
    struct.pack_into("<fiiii", buf, 44, hdr["dt_default"], hdr["fps"], hdr["rank"], hdr["world"], hdr["error"])
    struct.pack_into("<ffffdqq", buf, 64, hdr["dt"], hdr["next_dt"], hdr["step_time"], hdr["frame_time"], hdr["sim_time"], hdr["steps"], hdr["frames"])
    struct.pack_into("<iiii", buf, 104, hdr["pbc"], hdr["nbc"], hdr["ebc"], hdr["max_blocks"])
    struct.pack_into("<QQQQ", buf, 120, hdr["keys_offset"], hdr["keys_bytes"], hdr["grid_offset"], hdr["grid_bytes"])
    for i, e in enumerate(toc):
        struct.pack_into("<iiqQQ", buf, 256 + TOC * i, e["material"], e["channels"], e["count"], e["offset"], e["bytes"])
        struct.pack_into(PARAM_FMT, buf, 256 + TOC * i + 32, *_params(i))
    for e, st in zip(toc, states):   # the data where the unedited layout put it
        o = e["offset"]
        if o + st.nbytes <= len(buf) and o >= HEADER:
            buf[o: o + st.nbytes] = st.tobytes()
    if keys_off + keys.nbytes <= len(buf):
        buf[keys_off: keys_off + keys.nbytes] = keys.tobytes()
    if grid_off + grid.nbytes <= len(buf):
        buf[grid_off: grid_off + grid.nbytes] = grid.tobytes()
    return bytes(buf), dict(states=states, keys=keys, grid=grid, clock=c, cfg=cfg, toc=toc, keys_offset=keys_off, grid_offset=grid_off)


def _inspect(blob):
    from claymore_b200 import _capi
    inf = _capi.CheckpointInfo()
    arr = np.frombuffer(blob, np.uint8) if len(blob) else np.zeros(1, np.uint8)
    return _capi.lib().cb200_checkpoint_inspect(arr.ctypes.data_as(C.c_void_p), len(blob), C.byref(inf)), inf


def test_info_struct_matches_the_c_layout(tmp_path):
    from claymore_b200 import _capi
    M, I = _capi.CheckpointModel, _capi.CheckpointInfo
    fields = ["version", "n_models", "bytes", "cfg", "dt_default", "fps", "error", "dt", "sim_time", "steps", "frames", "particle_block_count",
              "max_blocks", "keys_offset", "grid_bytes", "models"]
    mfields = ["material", "channels", "count", "offset", "bytes", "params"]
    prog = ['#include <stdio.h>', '#include <stddef.h>', '#include "claymore_b200.h"', "int main(){",
            'printf("%zu %zu\\n", sizeof(cb200_checkpoint_info), sizeof(cb200_checkpoint_model));']
    prog += [f'printf("%zu\\n", offsetof(cb200_checkpoint_info, {f}));' for f in fields]
    prog += [f'printf("%zu\\n", offsetof(cb200_checkpoint_model, {f}));' for f in mfields]
    prog += ['printf("%d %d\\n", CB200_CHECKPOINT_VERSION, CB200_CHECKPOINT_HEADER_BYTES);', "return 0;}"]
    (tmp_path / "t.c").write_text("\n".join(prog) + "\n")
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), "-o", str(tmp_path / "t"), str(tmp_path / "t.c")])
    out = [int(x) for x in subprocess.check_output([str(tmp_path / "t")]).split()]
    assert out[:2] == [C.sizeof(I), C.sizeof(M)]
    assert out[2: 2 + len(fields)] == [getattr(I, f).offset for f in fields]
    assert out[2 + len(fields): -2] == [getattr(M, f).offset for f in mfields]
    assert out[-2:] == [_capi.CHECKPOINT_VERSION, _capi.CHECKPOINT_HEADER_BYTES]


def test_written_blob_is_accepted_and_read_bit_identically(tmp_path):
    from claymore_b200 import checkpoint
    blob, ref = make_blob()
    err, inf = _inspect(blob)
    assert err == 0
    c = ref["clock"]
    assert (inf.version, inf.n_models, inf.bytes) == (1, 2, len(blob))
    assert (inf.cfg.domain_bits, inf.cfg.max_ppc, inf.cfg.boundary) == ref["cfg"][:3]
    assert inf.cfg.gravity == np.float32(-9.8) and inf.cfg.cfl == np.float32(0.5)
    assert (inf.dt_default, inf.fps, inf.mgsp_rank, inf.mgsp_world, inf.error) == (np.float32(1e-4), 24, 0, 1, 0)
    assert (inf.dt, inf.next_dt, inf.step_time, inf.frame_time) == tuple(np.float32(c[k]) for k in ("dt", "next_dt", "step_time", "frame_time"))
    assert (inf.sim_time, inf.steps, inf.frames) == (c["sim_time"], c["steps"], c["frames"])
    assert (inf.particle_block_count, inf.neighbor_block_count, inf.exterior_block_count, inf.max_blocks) == (c["pbc"], c["nbc"], c["ebc"], c["max_blocks"])
    assert (inf.keys_offset, inf.grid_offset, inf.keys_bytes, inf.grid_bytes) == (ref["keys_offset"], ref["grid_offset"], 40 * 12, 40 * 1024)
    for i, e in enumerate(ref["toc"]):
        m = inf.models[i]
        assert (m.material, m.channels, m.count, m.offset, m.bytes) == (e["material"], e["channels"], e["count"], e["offset"], e["bytes"])
        p = m.params
        got = (p.rho, p.volume, p.mass, p.bulk, p.gamma, p.viscosity, p.lambda_, p.mu, p.cohesion, p.beta, p.yield_surface, p.volume_correction,
               p.bm, p.xi, p.msqr, p.hardening_on)
        assert got == struct.unpack(PARAM_FMT, struct.pack(PARAM_FMT, *_params(i)))
        assert p.material == e["material"] and not p.bins
    path = tmp_path / "a.ckpt"
    path.write_bytes(blob)
    for src in (str(path), blob):
        d = checkpoint.read(src)
        assert len(d["states"]) == 2
        for a, b in zip(d["states"], ref["states"]):
            assert a.shape == b.shape and a.tobytes() == b.tobytes()
        assert d["keys"].tobytes() == ref["keys"].tobytes() and d["grid"].tobytes() == ref["grid"].tobytes()
        assert d["models"][1]["params"]["rho"] == np.float32(1001.0) and d["steps"] == c["steps"]
    assert checkpoint.info(str(path))["cfg"]["domain_bits"] == 6


def _rejected(blob):
    return _inspect(blob)[0] == 1   # cudaErrorInvalidValue


def test_truncation_at_every_section_boundary_is_rejected():
    blob, ref = make_blob()
    cuts = {0, 8, HEADER - 1, HEADER, len(blob) - 1}
    for e in ref["toc"]:
        cuts |= {e["offset"], e["offset"] + e["bytes"]}
    cuts |= {ref["keys_offset"], ref["keys_offset"] + 40 * 12, ref["grid_offset"]}
    for n in sorted(cuts):
        assert _rejected(blob[:n]), n
    assert _rejected(blob + b"\0")   # longer than the header says
    assert not _rejected(blob)


def _edit(**kw):
    def f(hdr, toc):
        for k, v in kw.items():
            if k.startswith("toc"):
                i, field = k[3], k[5:]
                toc[int(i)][field] = v(toc[int(i)][field]) if callable(v) else v
            else:
                hdr[k] = v(hdr[k]) if callable(v) else v
    return f


CORRUPTIONS = {
    "magic": _edit(magic=b"CB200CKQ"),
    "version": _edit(version=2),
    "no_models": _edit(n_models=0),
    "nine_models": _edit(n_models=9),
    "material": _edit(toc0_material=4),
    "negative_material": _edit(toc1_material=-1),
    "channels": _edit(toc0_channels=13),
    "count_vs_bytes": _edit(toc0_count=lambda n: n + 1),
    "negative_count": _edit(toc0_count=-300, toc0_bytes=0),
    "bytes_vs_count": _edit(toc1_bytes=lambda b: b - 4),
    "keys_bytes": _edit(keys_bytes=lambda b: b - 12),
    "grid_bytes": _edit(grid_bytes=lambda b: b + 1024),
    "model_overlaps_model": _edit(toc1_offset=lambda o: o - 256),
    "keys_overlap_grid": _edit(keys_offset=lambda o: o + 512),
    "model_in_header": _edit(toc0_offset=HEADER - 4),
    "past_end": _edit(toc1_offset=lambda o: o + (1 << 20)),
    "wrapping_offset": _edit(grid_offset=(1 << 64) - 512),
    "pbc_zero": _edit(pbc=0),
    "pbc_above_nbc": _edit(pbc=41),
    "nbc_above_ebc": _edit(ebc=39),
    "negative_ebc": _edit(ebc=-1),
    "world": _edit(world=0),
    "rank": _edit(rank=1),
}


@pytest.mark.parametrize("name", sorted(CORRUPTIONS))
def test_corrupted_header_is_rejected(name):
    blob, _ = make_blob(layout=CORRUPTIONS[name])
    assert _rejected(blob)


@pytest.mark.parametrize("axis", [0, 1, 2])
@pytest.mark.parametrize("value", [-1, 16])
def test_key_outside_the_domain_is_rejected(axis, value):
    blob, ref = make_blob()
    b = bytearray(blob)
    struct.pack_into("<i", b, ref["keys_offset"] + 12 * 7 + 4 * axis, value)
    assert _rejected(bytes(b))


def test_repeated_key_is_rejected():
    blob, ref = make_blob()
    b = bytearray(blob)
    o = ref["keys_offset"]
    b[o + 12 * 5: o + 12 * 6] = b[o + 12 * 2: o + 12 * 3]
    assert _rejected(bytes(b))


def test_bad_config_is_rejected():
    assert _rejected(make_blob(cfg=(6, 100, 2, -9.8, 0.5))[0])
    assert _rejected(make_blob(cfg=(12, 128, 2, -9.8, 0.5))[0])


def test_offsets_beyond_two_gib_are_64_bit(tmp_path):
    """A 45 M-particle fixed-corotated model is 2.16e9 bytes: the keys and grid sections lie past 2^31 in a sparse file."""
    from claymore_b200 import checkpoint
    n = 45_000_000
    nbc = 8
    model_bytes = n * 12 * 4
    assert model_bytes > 1 << 31
    keys_off = _align(HEADER + model_bytes)
    grid_off = _align(keys_off + nbc * 12)
    total = grid_off + nbc * 1024
    head, _ = make_blob(models=[(1, 1)], nbc=nbc, clock=dict(pbc=2), layout=_edit(toc0_count=n, toc0_bytes=model_bytes, keys_offset=keys_off, grid_offset=grid_off, bytes=total), header_only=True)
    keys = np.array([[1, 2, 3], [1, 2, 4], [2, 2, 3], [2, 2, 4], [1, 3, 3], [1, 3, 4], [2, 3, 3], [2, 3, 4]], "<i4")
    path = tmp_path / "big.ckpt"
    with open(path, "wb") as f:
        f.write(head[:HEADER])
        f.truncate(total)
        f.seek(keys_off)
        f.write(keys.tobytes())
        f.seek(grid_off)
        f.write(np.full((nbc, 256), 2.5, "<f4").tobytes())
    d = checkpoint.read(str(path))
    m = d["models"][0]
    assert (m["count"], m["offset"], m["bytes"]) == (n, HEADER, model_bytes)
    assert (d["keys_offset"], d["grid_offset"], d["bytes"]) == (keys_off, grid_off, total)
    assert d["keys_offset"] > 1 << 31
    assert d["states"][0].shape == (n, 12)
    assert np.array_equal(d["keys"], keys) and (d["grid"] == 2.5).all()
    del d


def test_scene_resume_rejects_another_config_before_creating_a_simulator(tmp_path, monkeypatch):
    from claymore_b200 import scene
    import claymore_b200 as cb
    blob, _ = make_blob(models=[(1, 300)], cfg=(6, 128, 2, -9.8, 0.5))
    path = tmp_path / "a.ckpt"
    path.write_bytes(blob)

    class NoSim(scene.GmpmSimulator):
        def __init__(self, *a, **k):
            raise AssertionError("a simulator was created")
    monkeypatch.setattr(scene, "GmpmSimulator", NoSim)
    doc = {"simulation": {"fps": 24, "default_dt": 1e-4}, "models": [{"constitutive": "fixed_corotated", "file": "box"}]}
    with pytest.raises(ValueError, match="config"):
        scene.parse_scene(doc, config=cb.Config(domain_bits=7), resume=str(path))
    with pytest.raises(ValueError, match="config"):
        scene.parse_scene(doc, config=cb.Config(domain_bits=6, cfl=0.4), resume=str(path))
    with pytest.raises(ValueError, match="fps"):
        scene.parse_scene(dict(doc, simulation={"fps": 30, "default_dt": 1e-4}), config=cb.Config(domain_bits=6), resume=str(path))
    with pytest.raises(ValueError, match="models"):
        scene.parse_scene(dict(doc, models=[{"constitutive": "jfluid"}]), config=cb.Config(domain_bits=6), resume=str(path))
    # the matching document gets as far as creating the simulator
    with pytest.raises(AssertionError, match="created"):
        scene.parse_scene(json.loads(json.dumps(doc)), config=cb.Config(domain_bits=6), resume=str(path))
