"""GPU tests of the signed-distance collider: the sm_90a kernels and the step driver against the CPU oracle.

Bounds, restated from test_gpu_parity's comparison: key sets per class (particle / neighbour / exterior) and block counts exact,
per-cell grid mass rel 1e-5 (+ abs floor 1e-5 * max), momentum abs 1e-4 * max|mv|, particle positions matched within 2e-6,
the rest of the particle state within 5e-5 (sand and NACC: 2e-4, their return mappings amplify the last-bit differences of the cells the
collider stops).  The kernel-level check is tighter: velocity per cell rel 1e-6 with an absolute floor
of 4e-6 * max|v| (1e-5 for a rotating collider; FMA contraction and the device's sinf / cosf), max |v|^2 rel 1e-6.
"""
import ctypes as C
import json
import threading

import numpy as np
import pytest

import collider_oracle_binding as cob
import oracle_binding as ob
import scenes
from claymore_b200 import levelset
from claymore_b200._capi import Collider, Config as EngineConfig, Partition

pytestmark = pytest.mark.gpu

TYPES = {"sticky": 0, "slip": 1, "separate": 2}


def _torch():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch


def _fields(domain_bits, shape):
    ecfg = EngineConfig(domain_bits=domain_bits)
    if shape == "sphere":
        return levelset.sphere(ecfg, (0.42, 0.30, 0.40), 0.09)
    if shape == "floor":
        return levelset.box(ecfg, (0.15, 0.15, 0.15), (0.85, 0.305, 0.85))
    return levelset.box(ecfg, (0.30, 0.20, 0.28), (0.47, 0.34, 0.49))


MOTIONS = {"static": {}, "trans_vel": {"trans_vel": (0.3, 0.5, -0.2)}, "omega": {"omega": (0.04, -0.07, 0.11)}, "dsdt": {"dsdt": 0.5}, "scale": {"scale": 1.1}}


def _params(typ, friction, motion):
    m = MOTIONS[motion]
    return dict(type=typ, friction=friction, trans=(0.0, 0.0, 0.0), trans_vel=m.get("trans_vel", (0, 0, 0)), omega=m.get("omega", (0, 0, 0)),
                scale=m.get("scale", 1.0), dsdt=m.get("dsdt", 0.0))


def _fill(col, p):
    col.rot_mat[:] = [1, 0, 0, 0, 1, 0, 0, 0, 1]
    col.trans[:], col.trans_vel[:], col.omega[:] = [float(v) for v in p["trans"]], [float(v) for v in p["trans_vel"]], [float(v) for v in p["omega"]]
    col.dsdt, col.scale, col.friction = float(p["dsdt"]), float(p["scale"]), float(p["friction"])
    col.type = TYPES[p["type"]] if isinstance(p["type"], str) else int(p["type"])
    return col


def _block_field(domain_bits, sdf, grad):
    g = 1 << (domain_bits - 2)
    a = np.concatenate([sdf[None], grad]).reshape(4, g, 4, g, 4, g, 4)
    return np.ascontiguousarray(a.transpose(1, 3, 5, 0, 2, 4, 6).reshape(-1)).astype(np.float32)


# ---- kernel level: cb200_update_grid_velocity_query_max_collider against orc_update_grid_velocity_query_max_collider ----------
@pytest.fixture(scope="module")
def start_grid(oracle):
    scene = scenes.small_cube()
    osim = scenes.build_oracle(ob, scene, sim_class=cob.ColliderOracleSim)
    _, nbc, _ = osim.block_counts()
    g0 = osim.grid_array(0)[: nbc * 256].copy()
    keys = osim.partition_arrays(0)["active_keys"][: nbc * 3].copy()
    cfg = ob.make_config(domain_bits=scene["domain_bits"])
    return cfg, nbc, g0, keys, osim.dt


def _engine_update(cuda_lib, cfg, nbc, g0, keys, dt, col, t):
    torch = _torch()
    t_g = torch.from_numpy(g0.copy()).cuda()
    t_k = torch.from_numpy(keys.copy()).cuda()
    t_mv = torch.zeros(1, dtype=torch.float32, device="cuda")
    part = Partition()
    part.active_keys = t_k.data_ptr()
    ecfg = EngineConfig(domain_bits=cfg.domain_bits, boundary=cfg.boundary)
    if col is None:
        e = cuda_lib.cb200_update_grid_velocity_query_max(C.byref(ecfg), nbc, C.c_void_p(t_g.data_ptr()), part, dt, C.c_void_p(t_mv.data_ptr()), None)
    else:
        e = cuda_lib.cb200_update_grid_velocity_query_max_collider(C.byref(ecfg), nbc, C.c_void_p(t_g.data_ptr()), part, dt, C.byref(col), t, C.c_void_p(t_mv.data_ptr()), None)
    assert e == 0
    torch.cuda.synchronize()
    return t_g.cpu().numpy(), float(t_mv.item())


@pytest.mark.parametrize("t", [0.0, 0.37])
@pytest.mark.parametrize("motion", sorted(MOTIONS))
@pytest.mark.parametrize("friction", [0.0, 0.3])
@pytest.mark.parametrize("typ", ["sticky", "slip", "separate"])
@pytest.mark.parametrize("shape", ["sphere", "box"])
def test_kernel_matches_oracle(oracle, cuda_lib, start_grid, shape, typ, friction, motion, t):
    torch = _torch()
    cfg, nbc, g0, keys, dt = start_grid
    sdf, grad = _fields(cfg.domain_bits, shape)
    field = _block_field(cfg.domain_bits, sdf, grad)
    p = _params(typ, friction, motion)
    # oracle
    ocol = _fill(cob.Collider(), p)
    ocol.sdf = field.ctypes.data
    og = g0.copy()
    part = ob.Partition()
    part.active_keys = keys.ctypes.data
    omv = np.zeros(1, np.float32)
    cob.lib().orc_update_grid_velocity_query_max_collider(C.byref(cfg), nbc, ob.ptr(og), part, dt, C.byref(ocol), t, ob.ptr(omv))
    # engine
    t_field = torch.from_numpy(field).cuda()
    ecol = _fill(Collider(), p)
    ecol.sdf = t_field.data_ptr()
    eg, emv = _engine_update(cuda_lib, cfg, nbc, g0, keys, dt, ecol, t)
    ov, ev = og.reshape(nbc, 4, 64)[:, 1:], eg.reshape(nbc, 4, 64)[:, 1:]
    # the device's FMA contraction and, for a rotating collider, its sinf / cosf move the material-space point by an ulp; where the
    # level set's gradient turns within a cell (a box's edges) the normal moves by up to 1/dx times that, and the slip / separate
    # projection carries it into every component
    floor = (1e-5 if motion == "omega" else 4e-6) * max(1.0, np.abs(ov).max())
    assert np.allclose(ev, ov, rtol=1e-6, atol=floor), f"max velocity difference {np.abs(ev - ov).max():.3e}"
    assert abs(emv - float(omv[0])) <= 1e-6 * max(1.0, float(omv[0]))
    # the collider acts on this grid
    plain = g0.copy()
    mv0 = np.zeros(1, np.float32)
    ob.lib().orc_update_grid_velocity_query_max(C.byref(cfg), nbc, ob.ptr(plain), part, dt, ob.ptr(mv0))
    assert not np.array_equal(plain, og)


def test_kernel_wall_band_cells_equal_no_collider(oracle, cuda_lib):
    """A field that is solid everywhere: cells whose node lies in the wall band keep the no-collider result, every other cell with
    mass is stopped (STICKY)."""
    torch = _torch()
    scene = scenes.small_cube(lo=4, hi=14, v0=(0.2, -0.5, 0.1))   # reaches into the wall band (2 blocks = 8 cells)
    osim = scenes.build_oracle(ob, scene, sim_class=cob.ColliderOracleSim)
    _, nbc, _ = osim.block_counts()
    g0 = osim.grid_array(0)[: nbc * 256].copy()
    keys = osim.partition_arrays(0)["active_keys"][: nbc * 3].copy()
    cfg = ob.make_config(domain_bits=scene["domain_bits"])
    N = 4 << (cfg.domain_bits - 2)
    sdf = -np.ones((N, N, N), np.float32)
    grad = np.zeros((3, N, N, N), np.float32)
    grad[1] = 1.0
    t_field = torch.from_numpy(_block_field(cfg.domain_bits, sdf, grad)).cuda()
    col = _fill(Collider(), _params("sticky", 0.3, "static"))
    col.sdf = t_field.data_ptr()
    eg, _ = _engine_update(cuda_lib, cfg, nbc, g0, keys, osim.dt, col, 0.0)
    pg, _ = _engine_update(cuda_lib, cfg, nbc, g0, keys, osim.dt, None, 0.0)
    eg, pg = eg.reshape(nbc, 4, 64), pg.reshape(nbc, 4, 64)
    G = 1 << (cfg.domain_bits - 2)
    k = keys.reshape(-1, 3)
    band = ((k < cfg.boundary) | (k >= G - cfg.boundary)).any(1)
    has_mass = (g0.reshape(nbc, 4, 64)[:, 0] > 0)
    assert (band[:, None] & has_mass).any() and (~band[:, None] & has_mass).any()
    assert np.array_equal(eg[band], pg[band])
    assert (eg[~band][:, 1:][np.broadcast_to(has_mass[~band][:, None, :], eg[~band][:, 1:].shape)] == 0).all()


# ---- step driver against the oracle -------------------------------------------------------------------------------------------
def _compare_state(osim, esim, label, pos_tol=2e-6, f_tol=5e-5):
    st = esim.stats()
    assert st.error == 0, (label, st.error)
    opb, onb, oeb = osim.block_counts()
    assert (st.particle_block_count, st.neighbor_block_count, st.exterior_block_count) == (opb, onb, oeb), label
    okeys, ekeys = osim.active_keys(), esim.active_keys()
    for lo, hi in ((0, opb), (opb, onb), (onb, oeb)):
        assert np.array_equal(np.sort(scenes.key_hash(okeys[lo:hi])), np.sort(scenes.key_hash(ekeys[lo:hi]))), (label, lo, hi)
    oh, og = scenes.grid_by_key(okeys, osim.grid())
    eh, eg = scenes.grid_by_key(ekeys, esim.grid())
    assert np.array_equal(oh, eh)
    assert np.allclose(eg[:, 0], og[:, 0], rtol=1e-5, atol=1e-5 * og[:, 0].max()), label
    scale = np.abs(og[:, 1:]).max()
    assert np.abs(eg[:, 1:] - og[:, 1:]).max() <= 1e-4 * scale, (label, np.abs(eg[:, 1:] - og[:, 1:]).max(), scale)
    for m in range(len(osim.counts)):
        so, se = osim.particle_state(m), esim.particle_state(m)
        assert len(so) == len(se), label
        idx = scenes.match_particles(so, se, tol=pos_tol)
        if so.shape[1] > 3:
            assert np.abs(se[idx][:, 3:] - so[:, 3:]).max() <= f_tol, label


def _set_both(osim, esim, domain_bits, shape, p):
    sdf, grad = _fields(domain_bits, shape)
    osim.set_collider(_fill(cob.Collider(), p), sdf, grad)
    esim.set_collider(sdf, grad, **p)
    return sdf, grad


@pytest.mark.timeout(600)
@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
@pytest.mark.parametrize("typ", ["sticky", "slip", "separate"])
@pytest.mark.parametrize("material", [scenes.FIXED_COROTATED, scenes.J_FLUID, scenes.SAND, scenes.NACC])
def test_cube_on_box_collider_matches_oracle(oracle, cuda_lib, material, typ, use_graph):
    scene = scenes.small_cube(material=material, v0=(0.3, -1.5, 0.2))
    osim = scenes.build_oracle(ob, scene, sim_class=cob.ColliderOracleSim)
    esim = scenes.build_engine(scene, use_graph=use_graph)
    _set_both(osim, esim, scene["domain_bits"], "floor", _params(typ, 0.3, "static"))
    for k in range(4):
        osim.step(10)
        esim.step(10)
        _compare_state(osim, esim, f"{typ} after {10 * (k + 1)} sub-steps", f_tol=2e-4 if material in (scenes.SAND, scenes.NACC) else 5e-5)
    # the floor held the cube up: no particle below its top by more than one cell
    assert esim.retrieve(0)[:, 1].min() >= 0.305 - 1.0 / 64
    assert esim.sim_time() == pytest.approx(osim.sim_time, rel=1e-6)
    esim.close()


@pytest.mark.timeout(600)
def test_fluid_dam_with_moving_paddle_matches_oracle(oracle, cuda_lib):
    scene = scenes.small_cube(material=scenes.J_FLUID, lo=18, hi=34, v0=(0.0, 0.0, 0.0))
    osim = scenes.build_oracle(ob, scene, sim_class=cob.ColliderOracleSim)
    esim = scenes.build_engine(scene)
    p = dict(_params("slip", 0.0, "static"), trans=(-0.08, 0.0, 0.0), trans_vel=(1.5, 0.0, 0.0))
    _set_both(osim, esim, scene["domain_bits"], "box", p)
    for k in range(4):
        osim.step(10)
        esim.step(10)
        _compare_state(osim, esim, f"paddle after {10 * (k + 1)} sub-steps")
    esim.close()


@pytest.mark.timeout(600)
@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
def test_set_and_clear_between_substeps(oracle, cuda_lib, use_graph):
    scene = scenes.small_cube(v0=(0.3, -1.5, 0.2))
    osim = scenes.build_oracle(ob, scene, sim_class=cob.ColliderOracleSim)
    esim = scenes.build_engine(scene, use_graph=use_graph)
    osim.step(10)
    esim.step(10)
    p = _params("sticky", 0.3, "trans_vel")
    _set_both(osim, esim, scene["domain_bits"], "floor", p)
    osim.step(10)
    esim.step(10)
    _compare_state(osim, esim, "collider set")
    osim.clear_collider()
    esim.clear_collider()
    osim.step(10)
    esim.step(10)
    _compare_state(osim, esim, "collider cleared")
    _set_both(osim, esim, scene["domain_bits"], "sphere", _params("slip", 0.0, "static"))
    esim.set_collider(type="separate", friction=0.3)       # parameters only: the uploaded field stays
    osim.set_collider(_fill(cob.Collider(), _params("separate", 0.3, "static")))
    osim.step(10)
    esim.step(10)
    _compare_state(osim, esim, "collider set again")
    esim.close()


def test_far_collider_changes_nothing(cuda_lib):
    scene = scenes.small_cube(v0=(0.3, -1.0, 0.2))
    a = scenes.build_engine(scene)
    b = scenes.build_engine(scene)
    sdf, grad = levelset.sphere(EngineConfig(domain_bits=scene["domain_bits"]), (0.8, 0.8, 0.8), 0.05)
    b.set_collider(sdf, grad, type="sticky")
    a.step(30)
    b.step(30)
    _same_state(a, b)
    a.close()
    b.close()


def _same_state(a, b):
    """two engine runs: the same blocks; grid and particles equal up to the order of the atomic sums"""
    ka, kb = a.active_keys(), b.active_keys()
    assert np.array_equal(np.sort(scenes.key_hash(ka)), np.sort(scenes.key_hash(kb)))
    ha, ga = scenes.grid_by_key(ka, a.grid())
    hb, gb = scenes.grid_by_key(kb, b.grid())
    assert np.array_equal(ha, hb)
    assert np.allclose(gb, ga, rtol=1e-5, atol=1e-6 * np.abs(ga).max())
    pa, pb = a.particle_state(0), b.particle_state(0)
    idx = scenes.match_particles(pa, pb, tol=1e-6)
    assert np.allclose(pb[idx], pa, rtol=0, atol=1e-5)


@pytest.mark.timeout(300)
def test_mgsp_two_ranks_sticky_floor_match_single_domain(oracle, cuda_lib):
    """The max |v|^2 the ranks agree on comes from the carry kernel's predictor: with a collider it must apply the collider, or dt
    (which the max drives here) departs from the single-domain oracle's."""
    from claymore_b200 import mgsp
    scene = scenes.small_cube(v0=(1.0, -10.0, 0.5))
    dt_default = 1e-3
    osim = scenes.build_oracle(ob, scene, dt=dt_default, sim_class=cob.ColliderOracleSim)
    p = _params("sticky", 0.3, "static")
    sdf, grad = _fields(scene["domain_bits"], "floor")
    osim.set_collider(_fill(cob.Collider(), p), sdf, grad)
    sims = []
    for r in range(2):
        sims.append(mgsp.build_rank_sim(mgsp.partition_scene(scene, r, 2), r, 2, dt_default, 4000, scenes.apply_material))
        sims[-1].set_collider(sdf, grad, **p)
    ptrs = [s.mgsp_inbox() for s in sims]
    for s in sims:
        s.mgsp_set_peers(ptrs)
    errs = []

    def run(fn):
        def go(s):
            try:
                fn(s)
            except Exception as e:  # pragma: no cover
                errs.append(e)
        th = [threading.Thread(target=go, args=(s,)) for s in sims]
        [t.start() for t in th]
        [t.join(120) for t in th]
        assert not errs and not any(t.is_alive() for t in th)
    run(lambda s: s.initial_setup())
    for k in range(4):
        osim.step(5)
        run(lambda s: (s.step(5), s.sync()))
        for s in sims:
            st = s.stats()
            assert st.error == 0
            assert st.dt == pytest.approx(osim.dt, rel=1e-5), (k, st.dt, osim.dt)
        pos = np.concatenate([s.retrieve(0) for s in sims])
        opos = osim.retrieve(0)
        assert len(pos) == len(opos)
        scenes.match_particles(opos, pos, tol=2e-6)
    for s in sims:
        s.close()


def test_scene_json_collider_equals_api(cuda_lib, tmp_path):
    from claymore_b200 import scene as scene_mod
    doc = {"simulation": {"fps": 0, "default_dt": 1e-4},
           "models": [{"type": "particles", "constitutive": "fixed_corotated", "file": "box", "offset": [0.3125, 0.3125, 0.3125], "span": [0.1875, 0.1875, 0.1875],
                       "velocity": [0.3, -1.5, 0.2], "rho": 1000.0, "volume": 1.0 / 64 ** 3 / 8, "youngs_modulus": 5e3, "poisson_ratio": 0.4}],
           "collider": {"file": "box", "offset": [0.15, 0.15, 0.15], "span": [0.7, 0.155, 0.7], "type": "slip", "friction": 0.2, "velocity": [0.1, 0.0, 0.0]}}
    cfg = EngineConfig(domain_bits=6)
    a = scene_mod.parse_scene(doc, config=EngineConfig(domain_bits=6), max_blocks=4000)
    a.initial_setup()
    del doc["collider"]
    b = scene_mod.parse_scene(doc, config=EngineConfig(domain_bits=6), max_blocks=4000)
    sdf, grad = levelset.box(cfg, (0.15, 0.15, 0.15), (0.85, 0.305, 0.85))
    b.set_collider(sdf, grad, type="slip", friction=0.2, trans_vel=(0.1, 0.0, 0.0))
    b.initial_setup()
    a.step(30)
    b.step(30)
    _same_state(a, b)
    # and the floor acted
    c = scene_mod.parse_scene(doc, config=EngineConfig(domain_bits=6), max_blocks=4000)
    c.initial_setup()
    c.step(30)
    assert a.retrieve(0)[:, 1].min() > c.retrieve(0)[:, 1].min() + 1e-4
    for s in (a, b, c):
        s.close()
