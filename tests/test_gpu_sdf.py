"""Level-set particle sampling on the GPU (cb200_sample_sdf, cb200_sim_init_model_sdf, the scene front-end) against the float64
restatement tests/sdf_ref.py: rows bit for bit and in order, lattice mode against the existing samplers, random-mode counts, and
simulations built from level sets against the same scene built with init_model."""
import ctypes as C
import glob
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import scenes
import sdf_ref as R
import claymore_b200 as cb
from claymore_b200 import sdf
from claymore_b200._capi import SdfSampling

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(p for p in glob.glob(os.path.join(HERE, "golden", "ref_sdf_*.npz")) if "two_dragons" not in p)


def _ls(n, h, phi):
    return sdf.parse(R.text(n, h, phi))


# (name, level set, domain_bits, offset, span, ppc, seed)
def _matrix():
    out = []
    sph = R.sphere((17, 19, 21), 0.5, (4.0, 4.5, 5.0), 3.6)
    tor = R.torus((24, 14, 24), 0.25, (2.9, 1.6, 2.9), 1.8, 0.7)
    pla = R.plate((12, 12, 9), 0.5, 4)
    two = R.two_bodies((26, 14, 14), 0.5)
    neg = R.all_negative((5, 6, 7), 1.0)
    drg = R.dragonish()
    for ppc, seed in ((8, 0), (1, 3), (64, 2**40 + 5)):
        out.append((f"sphere_ppc{ppc}", sph, 7, (0.2, 0.25, 0.3), (0.4, 0.4, 0.4), ppc, seed))
    out.append(("sphere_spc_below_1", sph, 6, (0.1, 0.1, 0.1), (0.12, 0.12, 0.12), 8, 9))     # c < dx / 2: spc < 1
    out.append(("torus", tor, 7, (0.3, 0.3, 0.3), (0.5, 0.5, 0.5), 8, 1))
    out.append(("plate", pla, 7, (0.2, 0.2, 0.2), (0.3, 0.3, 0.3), 27, 4))
    out.append(("two_bodies", two, 7, (0.05, 0.3, 0.3), (0.9, 0.9, 0.9), 8, 5))
    out.append(("all_negative_faces", neg, 6, (0.0, 0.0, 0.0), (1.0, 1.0, 1.0), 8, 6))       # B = [0, 1] on x (c = 1/6)
    out.append(("dragonish", drg, 7, (0.3, 0.2, 0.05), (0.9, 0.9, 0.9), 8, 7))
    out.append(("dragonish_z_faces", drg, 7, (0.3, 0.2, 0.0), (1.0, 1.0, 1.0), 8, 8))     # z: B = [0, 1] exactly
    return out


MATRIX = _matrix()


def _device(ls, cfg, offset, span, ppc, mode, seed):
    return sdf.sample(ls, cfg, offset, span, ppc=ppc, mode=mode, seed=seed)


@pytest.mark.parametrize("case", MATRIX, ids=[c[0] for c in MATRIX])
def test_random_rows_bitwise(case):
    name, (n, h, phi), bits, off, span, ppc, seed = case
    cfg = cb.Config(domain_bits=bits)
    got = _device(_ls(n, h, phi), cfg, off, span, ppc, "random", seed)
    want = R.sample_random(n, h, phi, bits, off, span, ppc, seed)
    assert len(want) > 0 and got.shape == want.shape, (got.shape, want.shape)
    assert got.tobytes() == want.tobytes()


@pytest.mark.parametrize("case", MATRIX, ids=[c[0] for c in MATRIX])
@pytest.mark.parametrize("k", [1, 2, 3, 4])
def test_lattice_rows_bitwise(case, k):
    name, (n, h, phi), bits, off, span, _, _ = case
    cfg = cb.Config(domain_bits=bits)
    got = _device(_ls(n, h, phi), cfg, off, span, k ** 3, "lattice", 0)
    want = R.sample_lattice(n, h, phi, bits, off, span, k ** 3)
    assert got.shape == want.shape and got.tobytes() == want.tobytes()


def test_spc_range_of_matrix():
    spcs = [R.random_spc(c[1][0], c[1][1], c[2], c[3], c[4], c[5])[1] for c in MATRIX]
    assert min(spcs) < 1 and max(spcs) > 8


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[8:-4])
@pytest.mark.parametrize("mode", ["random", "lattice"])
def test_reference_fixtures_bitwise(path, mode):
    f = dict(np.load(path))
    ls = sdf.parse(f["text"].tobytes())
    n, h, phi = ls.n, ls.h, ls.phi
    off, span = (0.2, 0.2, 0.2), (0.6, 0.6, 0.6)
    got = _device(ls, cb.Config(domain_bits=7), off, span, 8, mode, 3)
    want = (R.sample_random(n, h, phi, 7, off, span, 8, 3) if mode == "random" else R.sample_lattice(n, h, phi, 7, off, span, 8))
    assert got.tobytes() == want.tobytes()


def test_lattice_box_is_uniform_box():
    dx = 1.0 / 64
    n, h, phi = R.box((11, 9, 13), 0.5, (1.0, 1.0, 1.0), (4.0, 3.0, 5.0))
    off = 0.25 - 0.5 * dx
    got = _device(_ls(n, h, phi), cb.Config(domain_bits=6), (off,) * 3, (20 * dx, 16 * dx, 24 * dx), 8, "lattice", 0)
    assert got.tobytes() == cb.samplers.uniform_box(dx, [20, 20, 20], [32, 28, 36]).tobytes()


def test_lattice_sphere_is_samplers_sphere():
    bits, center, radius = 7, np.array([0.45, 0.5, 0.55]), 0.2
    dx = 1.0 / (1 << bits)
    hl = dx  # level-set nodes on the simulation nodes
    m = int(np.ceil((radius + 3 * dx) / hl))
    n = (2 * m + 1,) * 3
    origin = center - m * hl
    _, _, phi = R.sphere(n, hl, center - origin, radius)
    got = _device(_ls(n, hl, phi), cb.Config(domain_bits=bits), origin, (2 * m * hl,) * 3, 8, "lattice", 0)
    want = cb.samplers.sphere(dx, center, radius)
    # equal except within the trilinear interpolation error of the surface (phi is exact at the nodes; curvature error < dx^2 / r)
    band = dx * dx / radius
    d = lambda p: np.linalg.norm(p.astype(np.float64) - center, axis=1) - radius
    key = lambda p: set(map(bytes, p.view(np.uint8).reshape(len(p), 12)))
    gs, ws = key(got), key(want)
    only = [np.frombuffer(b, np.float32) for b in gs ^ ws]
    assert all(abs(d(p[None])[0]) <= band for p in only), max(abs(d(p[None])[0]) for p in only)
    assert len(only) < 0.01 * len(want)


@pytest.mark.parametrize("case", [MATRIX[0], MATRIX[4], MATRIX[6], MATRIX[8]], ids=lambda c: c[0])
def test_random_counts_within_5_sigma(case):
    name, (n, h, phi), bits, off, span, ppc, seed = case
    c, spc = R.random_spc(n, h, bits, off, span, ppc)
    got = _device(_ls(n, h, phi), cb.Config(domain_bits=bits), off, span, ppc, "random", seed)
    dx = 1.0 / (1 << bits)
    # V_neg in float64: the negative fraction of every valid cell on a 16^3 midpoint grid
    valid = R.valid_cells(n, phi)
    t = (np.arange(16) + 0.5) / 16
    sub = np.stack(np.meshgrid(t, t, t, indexing="ij"), -1).reshape(-1, 3)
    cells = np.stack([valid % (n[0] - 1), (valid // (n[0] - 1)) % (n[1] - 1), valid // ((n[0] - 1) * (n[1] - 1))], 1).astype(np.float64)
    frac = np.empty(len(valid))
    for i0 in range(0, len(valid), 512):
        q = (cells[i0:i0 + 512, None, :] + sub[None]).reshape(-1, 3)
        frac[i0:i0 + 512] = (R.trilinear(n, phi, q[:, 0], q[:, 1], q[:, 2]) < 0).reshape(-1, len(sub)).mean(1)
    split = (n[0] - 1) // 2   # two coarse regions along x, on a cell boundary
    region = (cells[:, 0] >= split).astype(int)
    gq = (got.astype(np.float64) - np.asarray(off)) / c
    gregion = (np.floor(gq[:, 0]) >= split).astype(int)
    n_cand = np.floor(len(valid) * spc)
    for sel, count in [(np.ones(len(valid), bool), len(got))] + [(region == r, int((gregion == r).sum())) for r in (0, 1)]:
        v_neg = frac[sel].sum() * c ** 3
        expect = ppc * v_neg / dx ** 3
        p = min(max(frac[sel].mean(), 1e-9), 1 - 1e-9)
        sigma = np.sqrt(n_cand * sel.mean() * p * (1 - p)) + 1.0
        assert abs(count - expect) <= 5 * sigma, (name, count, expect, sigma)


def test_repeatable_and_seeded():
    name, (n, h, phi), bits, off, span, ppc, _ = MATRIX[0]
    ls, cfg = _ls(n, h, phi), cb.Config(domain_bits=bits)
    a = _device(ls, cfg, off, span, ppc, "random", 1)
    b = _device(ls, cfg, off, span, ppc, "random", 1)
    c = _device(ls, cfg, off, span, ppc, "random", 2)
    assert a.tobytes() == b.tobytes()
    assert len(a) != len(c) or a.tobytes() != c.tobytes()
    assert not np.array_equal(a[: min(len(a), len(c))], c[: min(len(a), len(c))])


def _sorted_rows(x):
    return np.sort(np.ascontiguousarray(x).view(np.dtype((np.void, x.dtype.itemsize * x.shape[1]))).reshape(-1))


@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
def test_init_model_sdf_matches_init_model(use_graph):
    bits = 6
    cfg = cb.Config(domain_bits=bits)
    sph = R.sphere((13, 13, 13), 0.5, (3.0, 3.0, 3.0), 2.4)
    tor = R.torus((20, 12, 20), 0.25, (2.4, 1.4, 2.4), 1.5, 0.6)
    models = [(cb.FIXED_COROTATED, _ls(*sph), (0.3, 0.3, 0.3), (0.3, 0.3, 0.3), 8, "random", 4, (0.5, -0.5, 0.0)),
              (cb.J_FLUID, _ls(*tor), (0.35, 0.6, 0.3), (0.3, 0.3, 0.3), 8, "lattice", 0, (0.0, -1.0, 0.0)),
              (cb.SAND, _ls(*sph), (0.55, 0.25, 0.55), (0.2, 0.2, 0.2), 27, "lattice", 0, (0.0, 0.0, 0.0))]
    a = cb.GmpmSimulator(config=cfg, use_graph=use_graph, max_blocks=4000)
    b = cb.GmpmSimulator(config=cfg, use_graph=use_graph, max_blocks=4000)
    for mat, ls, off, span, ppc, mode, seed, v0 in models:
        host = sdf.sample(ls, cfg, off, span, ppc=ppc, mode=mode, seed=seed)
        a.init_model_sdf(mat, ls, off, span, v0, ppc=ppc, mode=mode, seed=seed)
        b.init_model(mat, host, v0)
        assert a.counts[-1] == len(host)
    a.initial_setup()
    b.initial_setup()
    for m in range(len(models)):
        assert _sorted_rows(a.particle_state(m)).tobytes() == _sorted_rows(b.particle_state(m)).tobytes()
    a.step(10)
    b.step(10)
    sa, sb = a.stats(), b.stats()
    assert sa.error == 0 and sb.error == 0 and sa.dt == sb.dt
    for m in range(len(models)):
        pa, pb = a.particle_state(m), b.particle_state(m)
        idx = scenes.match_particles(pb, pa, tol=2e-6)
        assert np.abs(pa[idx][:, 3:] - pb[:, 3:]).max() <= 5e-5
    a.close()
    b.close()


def test_rejections_leave_simulator_usable():
    cfg = cb.Config(domain_bits=6)
    n, h, phi = R.sphere((9, 9, 9), 0.5, (2.0, 2.0, 2.0), 1.5)
    ls = _ls(n, h, phi)
    pos_ls = _ls(*R.sphere((9, 9, 9), 0.5, (2.0, 2.0, 2.0), -1.0))   # phi > 0 everywhere: count 0
    sim = cb.GmpmSimulator(config=cfg, max_blocks=2000)
    L = cb.lib()
    good = dict(offset=(0.3, 0.3, 0.3), span=(0.3, 0.3, 0.3))

    def raw(material=cb.FIXED_COROTATED, level=ls, mode=0, ppc=8, offset=good["offset"], span=good["span"]):
        smp = SdfSampling()
        smp.mode, smp.ppc, smp.seed = mode, ppc, 0
        smp.offset[:], smp.span[:] = offset, span
        ph = np.ascontiguousarray(level.phi)
        mid, cnt = C.c_int(-1), C.c_int(0)
        return L.cb200_sim_init_model_sdf(sim.h, material, C.byref(level.header), ph.ctypes.data_as(C.c_void_p), C.byref(smp), None,
                                          C.byref(mid), C.byref(cnt))

    bad = [dict(material=4), dict(material=-1), dict(mode=2), dict(ppc=0), dict(ppc=-8), dict(mode=1, ppc=9), dict(mode=1, ppc=125),
           dict(span=(0.3, 0.0, 0.3)), dict(span=(-0.3, 0.3, 0.3)), dict(offset=(-0.01, 0.3, 0.3)), dict(offset=(0.8, 0.3, 0.3)),
           dict(level=pos_ls)]
    for kw in bad:
        assert raw(**kw) == 1, kw   # cudaErrorInvalidValue
    assert len(sim.materials) == 0
    with pytest.raises(ValueError):
        sim.init_model_sdf(cb.FIXED_COROTATED, ls, (0.8, 0.3, 0.3), 0.3)
    for _ in range(8):
        sim.init_model_sdf(cb.FIXED_COROTATED, ls, good["offset"], good["span"], ppc=1)
    assert raw() == 1   # a ninth model
    sim.initial_setup()
    assert raw() == 1   # set up already
    sim.step(3)
    assert sim.stats().error == 0
    sim.close()
    sim = cb.GmpmSimulator(config=cfg, max_blocks=2000)
    sim.init_model_sdf(cb.FIXED_COROTATED, ls, good["offset"], good["span"])
    sim.initial_setup()
    sim.step(3)
    assert sim.stats().error == 0
    sim.close()


def _scene_doc(sdf_name, extra):
    m = {"type": "particle", "file": sdf_name, "constitutive": "jfluid", "volume": 7.45e-9, "rho": 1e3, "bulk_modulus": 4e4, "gamma": 7.15,
         "viscosity": 0.01, "offset": [0.3, 0.2, 0.05], "span": [0.9, 0.9, 0.9], "velocity": [0.0, -1.0, 0.0]}
    m.update(extra)
    return {"simulation": {"gpuid": 0, "fps": 1200, "frames": 1, "default_dt": 5e-6}, "models": [m]}


@pytest.mark.parametrize("extra", [{}, {"sampler": "lattice", "ppc": 27}, {"sampler": "random", "ppc": 4, "seed": 12345}],
                         ids=["defaults", "lattice27", "random_seeded"])
def test_scene_sdf_model(tmp_path, extra):
    n, h, phi = R.dragonish()
    sub = tmp_path / "levelsets"
    sub.mkdir()
    (sub / "dragons.sdf").write_bytes(R.text(n, h, phi))
    (tmp_path / "scene.json").write_text(json.dumps(_scene_doc("levelsets/dragons.sdf", extra)))
    cfg = cb.Config(domain_bits=7)
    sim = cb.scene.parse_scene(str(tmp_path / "scene.json"), config=cfg, max_blocks=4000)
    mode, ppc, seed = extra.get("sampler", "random"), extra.get("ppc", 8), extra.get("seed", 0)
    want = (R.sample_random(n, h, phi, 7, (0.3, 0.2, 0.05), (0.9,) * 3, ppc, seed) if mode == "random"
            else R.sample_lattice(n, h, phi, 7, (0.3, 0.2, 0.05), (0.9,) * 3, ppc))
    assert sim.counts == [len(want)] and sim.materials == [cb.J_FLUID]
    sim.initial_setup()
    st = sim.particle_state(0)
    assert _sorted_rows(np.ascontiguousarray(st[:, :3])).tobytes() == _sorted_rows(want).tobytes()
    sim.close()


def test_scene_cli_one_frame(tmp_path):
    n, h, phi = R.dragonish()
    (tmp_path / "dragons.sdf").write_bytes(R.text(n, h, phi))
    doc = _scene_doc("dragons.sdf", {"offset": [0.3, 0.2, 0.05], "span": [0.6, 0.6, 0.6]})
    (tmp_path / "scene.json").write_text(json.dumps(doc))
    out = tmp_path / "frames"
    out.mkdir()
    root = os.path.dirname(HERE)
    r = subprocess.run([sys.executable, "-m", "claymore_b200", "-f", str(tmp_path / "scene.json"), "--out", str(out)], cwd=root,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    pts = cb.bgeo.read(str(out / "model_id[0]_frame[1].bgeo"))
    want = R.sample_random(n, h, phi, 8, (0.3, 0.2, 0.05), (0.6,) * 3, 8, 0)
    assert len(pts["position"]) == len(want)


def test_scale_two_spheres_512():
    """the bench scene's two spheres (radius 0.1645 at x = 0.3 / 0.7, 512^3) as level sets on the simulation nodes, lattice ppc 8"""
    bits, radius = 9, 0.1645
    dx = 1.0 / (1 << bits)
    cfg = cb.Config(domain_bits=bits)
    total = 0
    for cx in (0.30, 0.70):
        center = np.array([cx, 0.5, 0.5])
        m = int(np.ceil((radius + 3 * dx) / dx))
        n = (2 * m + 1,) * 3
        origin = center - m * dx
        _, _, phi = R.sphere(n, dx, center - origin, radius)
        ls = _ls(n, dx, phi)
        got = sdf.sample(ls, cfg, origin, (2 * m * dx,) * 3, ppc=8, mode="lattice")
        total += len(got)
        # the restatement's count: only points within 2 level-set cells of the surface need phi (elsewhere all corners agree)
        assert len(got) == _lattice_count_sphere(n, dx, phi, origin, m, bits, center, radius)
        # rows of seeded x-slabs, in order (x is the slowest axis, so a slab's rows are contiguous)
        rng = np.random.default_rng(int(cx * 10))
        cells_x = np.floor(got[:, 0].astype(np.float64) / dx + 0.5).astype(np.int64)
        for i in rng.integers(int((cx - radius) / dx), int((cx + radius) / dx), 3):
            want = R.sample_lattice(n, dx, phi, bits, origin, (2 * m * dx,) * 3, 8, x_slabs=(int(i), int(i) + 1))
            sel = np.flatnonzero(cells_x == i)
            assert sel.size == 0 or np.all(np.diff(sel) == 1)
            assert got[sel].tobytes() == want.tobytes()
    assert total > 39_000_000


def _lattice_count_sphere(n, h, phi, origin, m, bits, center, radius):
    dx = 1.0 / (1 << bits)
    count = 0
    a = (np.arange(2, dtype=np.float64) - 0.5) / 2
    offs = np.stack(np.meshgrid(a, a, a, indexing="ij"), -1).reshape(-1, 3)
    c = R.node_box(n, h, origin, (2 * m * h,) * 3)[0]
    lo = [max(0, int(np.floor(origin[d] / dx)) - 1) for d in range(3)]
    hi = [min(1 << bits, int(np.ceil((origin[d] + (n[d] - 1) * c) / dx)) + 2) for d in range(3)]
    j, k = np.meshgrid(np.arange(lo[1], hi[1]), np.arange(lo[2], hi[2]), indexing="ij")
    for i in range(lo[0], hi[0]):
        cl = np.stack([np.full_like(j, i), j, k], -1).reshape(-1, 1, 3).astype(np.float64)
        x = ((cl + offs[None]) * dx).reshape(-1, 3).astype(np.float32)
        q = (x.astype(np.float64) - origin) / c
        inside = np.all((q >= 0) & (q <= np.asarray(n, np.float64) - 1), 1)
        d = np.linalg.norm(x.astype(np.float64) - center, axis=1) - radius
        sure = inside & (d < -2 * h)
        unsure = inside & (np.abs(d) <= 2 * h)
        count += int(sure.sum())
        if unsure.any():
            qu = q[unsure]
            count += int((R.trilinear(n, phi, qu[:, 0], qu[:, 1], qu[:, 2]) < 0).sum())
    return count
