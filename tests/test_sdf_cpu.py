"""Level-set particle sampling without a GPU: the library's .sdf parser against the reference's LoadSDF (fixtures recorded by
tests/golden/make_ref_sdf_golden.py), its rejections, Philox's known answers, and the float64 restatement (tests/sdf_ref.py)
against the reference's GenerateUniformSamples: valid cells, sample sign and distribution."""
import ctypes as C
import glob
import json
import os

import numpy as np
import pytest
from scipy import stats

import sdf_ref as R
import claymore_b200 as cb
from claymore_b200 import sdf

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")
FIXTURES = sorted(p for p in glob.glob(os.path.join(GOLDEN, "ref_sdf_*.npz")) if "two_dragons" not in p)
DRAGONS_NPZ = os.path.join(GOLDEN, "ref_sdf_two_dragons.npz")
DRAGONS_SDF = os.path.join(os.environ.get("CLAYMORE_REFERENCE", "/root/reference"), "Data", "MpmParticles", "two_dragons.sdf")


def _fix(path):
    return dict(np.load(path))


def test_philox_known_answers():
    cases = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
             ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
             ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for ctr, key, want in cases:
        assert tuple(int(v) for v in R.philox4x32_10(np.array([ctr], np.uint32), key)[0]) == want


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[8:-4])
def test_parser_equals_reference_loadsdf(path):
    f = _fix(path)
    ls = sdf.parse(f["text"].tobytes())
    assert ls.n == tuple(int(v) for v in f["dims"])
    assert np.float32(ls.h).tobytes() == np.float32(f["h"]).tobytes()
    assert np.array(ls.header.min, np.float32).tobytes() == f["mins"].astype(np.float32).tobytes()
    assert ls.phi.tobytes() == f["phi"].tobytes()


@pytest.mark.skipif(not os.path.exists(DRAGONS_SDF), reason="the reference checkout with its Data/ is not here")
def test_parser_on_two_dragons():
    ls = sdf.read(DRAGONS_SDF)
    assert ls.n == (77, 118, 401) and ls.h == 0.25
    shim = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "libclaymore_ref_sdf.so")
    if os.path.exists(shim):
        L = C.CDLL(shim)
        dims, mins, h = np.zeros(3, np.int32), np.zeros(3, np.float32), np.zeros(1, np.float32)
        phi = np.zeros(ls.phi.size, np.float32)
        L.ref_sdf_load.argtypes = [C.c_char_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong]
        L.ref_sdf_load(DRAGONS_SDF.encode(), dims.ctypes.data, mins.ctypes.data, h.ctypes.data, phi.ctypes.data, phi.size)
        assert phi.tobytes() == ls.phi.tobytes()
    assert len(R.valid_cells(ls.n, ls.phi)) == 252867


def test_parser_round_trips_written_fields():
    n, h, phi = R.torus((7, 6, 9), 0.3, (1.0, 0.8, 1.2), 0.7, 0.3)
    ls = sdf.parse(R.text(n, h, phi))
    assert ls.phi.tobytes() == phi.tobytes() and ls.grid.shape == (9, 6, 7)
    ls2 = sdf.parse("2 2 2\n0 0 0\n1e-1\n" + " ".join(["-1.5e-45", "3.4028235e38", "-0", "1", "2", "3", "4", "5"]) + "  \n\n")
    assert ls2.phi.view(np.uint32)[:3].tolist() == [0x80000001, 0x7F7FFFFF, 0x80000000]


BAD = {
    "dimension below 2": "1 2 2\n0 0 0\n1\n" + "0 " * 4,
    "zero dimension": "0 2 2\n0 0 0\n1\n",
    "2^31 nodes": "1024 1024 2048\n0 0 0\n1\n0\n",
    "h zero": "2 2 2\n0 0 0\n0\n" + "0 " * 8,
    "h negative": "2 2 2\n0 0 0\n-1\n" + "0 " * 8,
    "h inf": "2 2 2\n0 0 0\ninf\n" + "0 " * 8,
    "h nan": "2 2 2\n0 0 0\nnan\n" + "0 " * 8,
    "value inf": "2 2 2\n0 0 0\n1\n" + "0 " * 7 + "inf",
    "value nan": "2 2 2\n0 0 0\n1\nnan " + "0 " * 7,
    "value overflows": "2 2 2\n0 0 0\n1\n1e39 " + "0 " * 7,
    "too few": "2 2 2\n0 0 0\n1\n" + "0 " * 7,
    "too many": "2 2 2\n0 0 0\n1\n" + "0 " * 9,
    "garbage value": "2 2 2\n0 0 0\n1\n" + "0 " * 7 + "x",
    "truncated header": "2 2",
    "empty": "",
}


@pytest.mark.parametrize("name", list(BAD))
def test_parser_rejections(name):
    text = BAD[name].encode()
    hdr = cb._capi.SdfHeader()
    assert cb.lib().cb200_sdf_parse(text, len(text), C.byref(hdr), None, 0) != 0
    with pytest.raises(ValueError):
        sdf.parse(text)


def test_parser_capacity_below_count():
    text = R.text(*R.sphere((3, 3, 3), 1.0, (1, 1, 1), 0.5))
    hdr, phi = cb._capi.SdfHeader(), np.zeros(27, np.float32)
    assert cb.lib().cb200_sdf_parse(text, len(text), C.byref(hdr), phi.ctypes.data_as(C.c_void_p), 26) != 0
    assert cb.lib().cb200_sdf_parse(text, len(text), C.byref(hdr), phi.ctypes.data_as(C.c_void_p), 27) == 0


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[8:-4])
def test_valid_cells_equal_reference(path):
    f = _fix(path)
    assert len(R.valid_cells(tuple(f["dims"]), f["phi"])) == int(f["V"])
    assert int(f["gmpm_sample_num"]) == int(np.float32(int(f["V"])) * (np.float32(8) * np.float32(int(f["dims"].min())) / np.float32(256)))


def test_two_dragons_counts():
    f = _fix(DRAGONS_NPZ)
    assert tuple(f["dims"]) == (77, 118, 401) and float(f["h"]) == 0.25
    assert int(f["V"]) == 252867 and int(f["gmpm_sample_num"]) == 608461
    assert int(f["hist"].sum()) == 608461


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[8:-4])
def test_reference_samples_are_inside(path):
    """every reference sample has phi < 0 under the float64 trilinear phi, outside a band of 1e-6 max|phi|"""
    f = _fix(path)
    n, phi = tuple(int(v) for v in f["dims"]), f["phi"]
    band = 1e-6 * float(np.abs(phi).max())
    for s in f["seeds"]:
        q = f[f"samples_{s}"].astype(np.float64)
        assert len(q) == int(int(f["V"]) * np.float32(f["spc"]))
        v = R.trilinear(n, phi, q[:, 0], q[:, 1], q[:, 2])
        assert np.all(v[np.abs(v) > band] < 0)


def _bin_counts(q, n, edges=4):
    bins = [np.arange(0, n[d] - 1 + edges, edges) for d in range(3)]
    return np.histogramdd(q, bins=bins)[0].reshape(-1)


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[8:-4])
def test_reference_distribution_matches_restatement(path):
    """S3's normalisation: the reference puts V spc samples into the negative region, the restatement keeps the thinned candidates;
    both are uniform over the negative region, so their 4^3-cell bin shares must agree (chi-square two-sample test)."""
    f = _fix(path)
    n, phi = tuple(int(v) for v in f["dims"]), f["phi"]
    ref = np.concatenate([f[f"samples_{s}"] for s in f["seeds"]]).astype(np.float64)
    ours = np.concatenate([q[k] for seed in (11, 12) for q, k in R.random_index_samples(n, phi, 16.0, seed)])
    a, b = _bin_counts(ref, n), _bin_counts(ours, n)
    m = (a + b) > 0
    p = stats.chi2_contingency(np.stack([a[m], b[m]]))[1]
    assert p > 1e-4, p
    # S3: the reference's density over the negative region is V / V_neg times the nominal one
    assert len(ours) / (2 * 16.0 * int(f["V"])) < 1.0


def test_scene_rejects_unfitted_box(tmp_path):
    """scene.json's placement (span 1 from offset 0.1) on a dragon-proportioned level set: rejected before any device work"""
    n, h, phi = R.dragonish()
    (tmp_path / "dragons.sdf").write_bytes(R.text(n, h, phi))
    doc = {"simulation": {"fps": 24, "frames": 1}, "models": [
        {"type": "particle", "file": "dragons.sdf", "constitutive": "jfluid", "volume": 7.45e-9, "rho": 1e3, "bulk_modulus": 4e4, "gamma": 7.15,
         "viscosity": 0.01, "offset": [0.1, 0.1, 0.1], "span": [1.0, 1.0, 1.0], "velocity": [0, -1, 0]}]}
    (tmp_path / "scene.json").write_text(json.dumps(doc))
    with pytest.raises(ValueError, match=r"model 0 \(dragons.sdf\): node box \[0.1, 0.1, 0.1\] - \[.*\] .*domain"):
        cb.scene.parse_scene(str(tmp_path / "scene.json"))
    doc["models"][0]["sampler"] = "poisson"
    doc["models"][0]["span"] = [0.2, 0.2, 0.2]
    (tmp_path / "scene.json").write_text(json.dumps(doc))
    with pytest.raises(ValueError, match="unknown sdf sampler"):
        cb.scene.parse_scene(str(tmp_path / "scene.json"))


def test_lattice_restatement_is_uniform_box():
    """k = 2 on a cell-aligned box: samplers.uniform_box's rows and bits"""
    dx = 1.0 / 64
    n, h, phi = R.box((11, 9, 13), 0.5, (1.0, 1.0, 1.0), (4.0, 3.0, 5.0))
    off = 0.25 - 0.5 * dx   # box faces half a cell below nodes: uniform_box's cells [lo, hi) span [lo - 1/2, hi - 1/2) dx
    span = (10 * 2 * dx, 8 * 2 * dx, 12 * 2 * dx)
    assert R.node_box(n, h, (off,) * 3, span)[0] == 2 * dx
    got = R.sample_lattice(n, h, phi, 6, (off,) * 3, span, 8)
    cell_lo, cell_hi = [20, 20, 20], [32, 28, 36]   # 16 + 2 (2 dx) per axis, to 16 + (8, 6, 10) (2 dx)
    want = cb.samplers.uniform_box(dx, cell_lo, cell_hi)
    assert got.tobytes() == want.tobytes()
