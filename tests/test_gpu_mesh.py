"""Level sets from triangle meshes on the device (claymore_b200.mesh, DESIGN.md section 2.12) against SDFGen itself.

phi and the header must equal SDFGen's make_level_set3 bit for bit: the recorded goldens (tests/golden/ref_sdfgen_*.npz: the torus
at three h, paddings 1 and 3, exact bands 0, 1 and 3; a cube on lattice nodes; an open box; two overlapping bodies; degenerate
triangles; a single triangle; a two-triangle floor 300 cells wide; unreferenced vertices) and, where oracle/_ref has the SDFGen
shim, live runs on further meshes.  Then the consumers: a model sampled from a mesh level set equals one sampled from its .sdf
round trip, a fluid block falling onto a torus obstacle built from the .obj follows the float64 reference, and a scene with .obj
model, boundary and sink equals the same API calls and resumes from a checkpoint.
"""
import glob
import json
import os

import numpy as np
import pytest

import mesh_cases as M
import ref64_cases as S
import ref64_levelset as RL
from claymore_b200 import _capi, mesh, objects, scene, sdf
from claymore_b200._capi import Config
from claymore_b200.simulator import GmpmSimulator
from ref64_checks import engine_substep_check

pytestmark = pytest.mark.gpu
GOLDENS = sorted(glob.glob(os.path.join(M.GOLDEN, "ref_sdfgen_*.npz")))
DOMAIN_BITS = 6
DX = 1.0 / 64


def _name(path):
    return os.path.basename(path)[len("ref_sdfgen_"):-len(".npz")]


def _assert_same(ls, dims, origin, h, phi, what):
    assert list(ls.n) == [int(x) for x in dims], what
    assert np.array_equal(np.asarray(ls.header.min[:], np.float32).view(np.uint32), np.asarray(origin, np.float32).view(np.uint32)), what
    assert np.float32(ls.h).view(np.uint32) == np.float32(h).view(np.uint32), what
    a, b = ls.phi.view(np.uint32), np.asarray(phi, np.float32).view(np.uint32)
    bad = np.flatnonzero(a != b)
    assert bad.size == 0, f"{what}: {bad.size} of {a.size} nodes differ, first {bad[:5]}: {ls.phi[bad[:5]]} vs {np.asarray(phi)[bad[:5]]}"


def test_goldens_exist():
    assert len(GOLDENS) == 12


@pytest.mark.parametrize("path", GOLDENS, ids=_name)
def test_golden_bitwise(cuda_lib, path):
    g = M.golden(path)
    ls = mesh.levelset(mesh.Mesh(g["vertices"], g["triangles"]), float(g["h"]), int(g["padding"]), int(g["exact_band"]))
    _assert_same(ls, g["dims"], g["origin"], g["h"], g["phi"], _name(path))


def _live_cases():
    tv, tt = M.torus()
    rng = np.random.default_rng(11)
    soup = (rng.random((60, 3)) * 2 - 1).astype(np.float32)
    rot = np.linalg.qr(rng.standard_normal((3, 3)))[0].astype(np.float32)
    return {"torus_h05_p2_b2": (tv, tt, 0.05, 2, 2), "torus_rotated_h04_b8": ((tv @ rot.T).astype(np.float32), tt, 0.04, 1, 8),
            "soup": (soup, rng.integers(0, 60, (40, 3)).astype(np.int32), 0.08, 1, 1),
            "cube_on_nodes_b0": M.cases()["cube_on_nodes"][:4] + (0,)}


@pytest.mark.parametrize("name", list(_live_cases()))
def test_live_sdfgen(cuda_lib, name):
    L = M.shim()
    if L is None:
        pytest.skip("oracle/_ref/libclaymore_ref_sdfgen.so not built (oracle/build_ref_sdfgen.sh)")
    v, t, h, padding, band = _live_cases()[name]
    n, lo, phi = M.ref_level_set(L, v, t, h, padding, band)
    _assert_same(mesh.levelset(mesh.Mesh(v, t), h, padding, band), n, lo, h, phi, name)


def test_two_builds_identical(cuda_lib):
    m = mesh.Mesh(*M.torus())
    a, b = mesh.levelset(m, 0.03, 2, 2), mesh.levelset(m, 0.03, 2, 2)
    assert np.array_equal(a.phi.view(np.uint32), b.phi.view(np.uint32))


def test_model_equals_sdf_round_trip(cuda_lib, tmp_path):
    ls = mesh.levelset(mesh.Mesh(*M.torus()), 0.04)
    sdf.write(ls, str(tmp_path / "torus.sdf"))
    back = sdf.read(str(tmp_path / "torus.sdf"))
    assert np.array_equal(back.phi.view(np.uint32), ls.phi.view(np.uint32))
    cfg = Config(domain_bits=DOMAIN_BITS)
    for mode, ppc in (("random", 8), ("lattice", 8)):
        a = sdf.sample(ls, cfg, (0.2, 0.3, 0.2), (0.6, 0.6, 0.6), ppc=ppc, mode=mode, seed=3)
        b = sdf.sample(back, cfg, (0.2, 0.3, 0.2), (0.6, 0.6, 0.6), ppc=ppc, mode=mode, seed=3)
        assert len(a) > 1000 and np.array_equal(a.view(np.uint32), b.view(np.uint32)), mode


@pytest.mark.timeout(900)
def test_fluid_onto_torus_from_obj_ref64(cuda_lib):
    """a fluid block falls onto a slip torus built from the .obj; 40 sub-steps against ref64 with test_gpu_levelset_ref64's bounds"""
    torus = mesh.levelset(mesh.Mesh(*M.torus()), 0.05)
    # node box x, z 0.35-0.65, y 0.25-0.36: the block (x, z 0.41-0.53, y from 0.375) lies over the ring and its hole
    obstacle = ("levelset", (torus, (0.35, 0.25, 0.35), (0.3, 0.3, 0.3)), dict(type=S.SLIP, friction=0.2))
    case = S._case(6, [S.model(S.J_FLUID, S.box(DX, (26, 24, 26), (34, 30, 34)), (0.0, -3.0, 0.0), DX)], [0, 5, 20, 39], dt=2e-4,
                   objects=[obstacle])
    with RL.registered([RL.lattice(torus.n, torus.phi)]):
        engine_substep_check(case, True, "fluid onto the .obj torus")


def _scene_files(tmp_path):
    M.write_torus_obj(tmp_path / "torus.obj")
    v, t = M.cube()
    (tmp_path / "cube.obj").write_text(M.plain_obj(v, t))
    return {"simulation": {"frames": 6, "fps": 120, "default_dt": 1e-3},
            "models": [{"constitutive": "fixed_corotated", "file": "cube.obj", "offset": [0.375, 0.5, 0.375], "span": [0.1875, 0.1875, 0.1875],
                        "velocity": [0, -1, 0], "rho": 1000, "volume": 1.0 / 64 ** 3 / 8, "youngs_modulus": 1e4, "poisson_ratio": 0.3,
                        "sampler": "lattice", "h": 0.05}],
            "boundaries": [{"shape": "levelset", "file": "torus.obj", "offset": [0.3, 0.3, 0.3], "span": [0.4, 0.4, 0.4], "type": "slip",
                            "friction": 0.2, "omega": [0, 0.5, 0]}],
            "sinks": [{"shape": "levelset", "file": "cube.obj", "offset": [0.3, 0.45, 0.3], "span": [0.15, 0.15, 0.15], "start": 2, "every": 2}]}


def test_scene_equals_api_calls(cuda_lib, tmp_path):
    from test_gpu_levelset_objects import _same_run
    doc = _scene_files(tmp_path)
    path = tmp_path / "scene.json"
    path.write_text(json.dumps(doc))
    cfg = Config(domain_bits=DOMAIN_BITS)
    a = scene.parse_scene(str(path), config=cfg, max_blocks=4000)
    a.main_loop()
    b = GmpmSimulator(dt=1e-3, fps=120, frames=6, config=cfg, max_blocks=4000)
    m = doc["models"][0]
    cube = mesh.read_obj(str(tmp_path / "cube.obj"))
    b.init_model_sdf(_capi.FIXED_COROTATED, mesh.levelset(cube, 0.05), m["offset"], m["span"], m["velocity"], ppc=8, mode="lattice")
    b.update_fr_parameters(m["rho"], m["volume"], m["youngs_modulus"], m["poisson_ratio"], model=0)
    torus = mesh.levelset(mesh.read_obj(str(tmp_path / "torus.obj")), a._levelsets[0].h)
    b.set_collision_objects([objects.levelset(torus, (0.3, 0.3, 0.3), (0.4, 0.4, 0.4), type="slip", friction=0.2, omega=(0, 0.5, 0))])
    # the sink's cube: default h = extent 1 x dx / 0.15
    sink = objects.levelset(mesh.levelset(cube, 1.0 * DX / 0.15), (0.3, 0.45, 0.3), (0.15, 0.15, 0.15))
    b.emitters = [lambda s, f: s.remove_particles([sink]) if f in (2, 4, 6) else None]
    b.main_loop()
    assert a.stats().error == 0 and b.stats().error == 0
    assert len(a._levelsets) == 2 and len(b._levelsets) == 2
    assert np.array_equal(a._levelsets[1].phi, sink.levelset.phi)
    _same_run(a, b)
    a.close(), b.close()


def test_scene_resume_equals_uninterrupted_run(cuda_lib, tmp_path):
    import test_gpu_collider as tgc
    doc = _scene_files(tmp_path)
    path = tmp_path / "scene.json"
    path.write_text(json.dumps(doc))
    cfg = Config(domain_bits=DOMAIN_BITS)
    ck = str(tmp_path / "f3.ckpt")
    a = scene.parse_scene(str(path), config=cfg, max_blocks=4000)
    seen = {}

    def on_frame(s, f):
        if f == 3:
            s.save_checkpoint(ck)
            seen["ok"] = True
    a.main_loop(on_frame=on_frame)
    assert a.stats().error == 0 and seen
    b = scene.parse_scene(str(path), config=cfg, max_blocks=4000, resume=ck)
    b.main_loop()
    assert b.stats().error == 0
    assert a.counts == b.counts
    tgc._same_state(a, b)
    a.close(), b.close()


def test_mesh2sdf_cli(cuda_lib, tmp_path):
    from claymore_b200.__main__ import main
    out = str(tmp_path / "t.sdf")
    assert main(["mesh2sdf", M.write_torus_obj(tmp_path / "t.obj"), out, "--h", "0.07"]) == 0
    g = M.golden(os.path.join(M.GOLDEN, "ref_sdfgen_torus_h07_p1_b1.npz"))
    _assert_same(sdf.read(out), g["dims"], g["origin"], g["h"], g["phi"], "mesh2sdf")
