"""GPU tests of the analytic collision objects (DESIGN.md section 2.9): the sm_90a grid update against the float64 reference
(ref64) per node and against the CPU oracle (oracle/collider_oracle.c), the objects entry with no objects against the existing
entries bit for bit, and the step driver and the MGSP predictors against the oracle with test_gpu_collider's bounds.

Kernel bounds: per node |v - ref| <= 1e-5 (1 + |v_ref|) (the device's sinf / cosf and FMA contraction), nodes near one of the
objects' discontinuities left out and counted (at most 2 %); the reported max |v|^2 is the max over the written velocities."""
import ctypes as C
import json

import numpy as np
import pytest

import threading

import collider_oracle_binding as cob
import oracle_binding as ob
import ref64
import scenes as ts
import test_gpu_collider as tgc
from claymore_b200 import _capi, levelset, objects, scenes
from claymore_b200._capi import Collider, CollisionObject, Config, Partition

pytestmark = pytest.mark.gpu
DOMAIN_BITS = 6


def _torch():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch


def _rot(ax, ay, az):
    cx, sx, cy, sy, cz, sz = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay), np.cos(az), np.sin(az)
    return np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]]) @ np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])


MOTIONS = {"static": {}, "combined": dict(rot=_rot(0.3, -0.2, 0.5), trans=(0.5, 0.47, 0.5), trans_vel=(0.04, -0.03, 0.02), omega=(0.3, -0.2, 0.5),
                                          scale=1.15, dsdt=0.2)}


def _shape(shape, **kw):
    if shape == "plane":
        return objects.plane((0.5, 0.45, 0.5), (0.3, 1.0, -0.2), **kw)
    if shape == "box":
        return objects.box((0.3, 0.28, 0.33), (0.68, 0.61, 0.7), **kw)
    if shape == "sphere":
        return objects.sphere((0.52, 0.47, 0.5), 0.21, **kw)
    return objects.cylinder((0.5, 0.5, 0.48), 0.18, 0.12, **kw)


@pytest.fixture(scope="module")
def grid():
    """every block of [2, 14)^3 on a 64^3 grid, masses log-uniform in [1e-3, 1] with some empty nodes, velocities N(0, 2)"""
    rng = np.random.default_rng(7)
    r = np.arange(2, 14)
    keys = np.stack(np.meshgrid(r, r, r, indexing="ij"), -1).reshape(-1, 3).astype(np.int32)
    nb = len(keys)
    g = np.zeros((nb, 4, 64), np.float32)
    m = np.exp(rng.uniform(np.log(1e-3), 0.0, (nb, 64))).astype(np.float32)
    m[rng.random((nb, 64)) < 0.05] = 0.0
    g[:, 0] = m
    g[:, 1:] = (rng.normal(0, 2.0, (nb, 3, 64)) * m[:, None]).astype(np.float32)
    return keys, g


def _run(cuda_lib, keys, g, dt, objs, t, col=None, entry="objects"):
    torch = _torch()
    t_g = torch.from_numpy(g.reshape(-1).copy()).cuda()
    t_k = torch.from_numpy(keys.reshape(-1).copy()).cuda()
    t_mv = torch.zeros(1, dtype=torch.float32, device="cuda")
    part = Partition()
    part.active_keys = t_k.data_ptr()
    cfg = Config(domain_bits=DOMAIN_BITS)
    arr = (CollisionObject * max(len(objs), 1))(*objs)
    G, MV = C.c_void_p(t_g.data_ptr()), C.c_void_p(t_mv.data_ptr())
    if entry == "plain":
        e = cuda_lib.cb200_update_grid_velocity_query_max(C.byref(cfg), len(keys), G, part, dt, MV, None)
    elif entry == "collider":
        e = cuda_lib.cb200_update_grid_velocity_query_max_collider(C.byref(cfg), len(keys), G, part, dt, C.byref(col), t, MV, None)
    else:
        e = cuda_lib.cb200_update_grid_velocity_query_max_objects(C.byref(cfg), len(keys), G, part, dt, C.byref(col) if col is not None else None, arr, len(objs), t, MV, None)
    assert e == 0
    torch.cuda.synchronize()
    return t_g.cpu().numpy().reshape(g.shape), float(t_mv.item())


def _check(cuda_lib, grid, objs, t, dt=1e-3):
    keys, g = grid
    eg, emx = _run(cuda_lib, keys, g, dt, objs, t)
    ref, _, _, info = ref64.grid_update(Config(domain_bits=DOMAIN_BITS), keys, g, dt, None, t, objects=objs)
    near = info["near"]
    has = g[:, 0] >= np.finfo(np.float32).tiny
    ok = has & ~near
    err = np.abs(eg[:, 1:] - ref).max(1)
    bound = 1e-5 * (1 + np.abs(ref).max(1))
    assert (err[ok] <= bound[ok]).all(), float((err[ok] / bound[ok]).max())
    assert near[has].mean() <= 0.02, near[has].mean()
    vsq = (eg[:, 1:].astype(np.float64) ** 2).sum(1)[has]
    assert emx == pytest.approx(vsq.max(), rel=1e-6)
    changed = (np.abs(ref - g[:, 1:] / np.where(has, g[:, 0], 1)[:, None]) > 0.0).any(1) & ok
    return ok.sum(), changed.sum()


@pytest.mark.parametrize("t", [0.0, 0.37, 3.1])
@pytest.mark.parametrize("motion", sorted(MOTIONS))
@pytest.mark.parametrize("friction", [0.0, 0.3])
@pytest.mark.parametrize("typ", ["sticky", "slip", "separate"])
@pytest.mark.parametrize("shape", ["plane", "box", "sphere", "cylinder"])
def test_kernel_matches_reference(cuda_lib, grid, shape, typ, friction, motion, t):
    kept, changed = _check(cuda_lib, grid, [_shape(shape, type=typ, friction=friction, **MOTIONS[motion])], np.float32(t))
    assert changed > 100, "the object must act on the grid"


@pytest.mark.parametrize("t", [0.0, 3.1])
def test_overlapping_objects_in_list_order(cuda_lib, grid, t):
    objs = [objects.sphere((0.5, 0.5, 0.5), 0.2, type="sticky", trans_vel=(0.1, 0.0, 0.0)),
            objects.box((0.4, 0.3, 0.35), (0.75, 0.6, 0.65), type="slip", friction=0.3, **MOTIONS["combined"]),
            objects.cylinder((0.45, 0.5, 0.5), 0.15, 0.2, type="separate", friction=0.0, omega=(0.0, 0.7, 0.0))]
    assert _check(cuda_lib, grid, objs, np.float32(t))[1] > 100
    # the order matters: the reversed list gives other velocities where the objects overlap
    keys, g = grid
    a, _ = _run(cuda_lib, keys, g, 1e-3, objs, np.float32(t))
    b, _ = _run(cuda_lib, keys, g, 1e-3, objs[::-1], np.float32(t))
    assert (a != b).any()


def test_no_objects_is_the_existing_entry_bit_for_bit(cuda_lib, grid):
    torch = _torch()
    keys, g = grid
    for t in (0.0, 0.37):
        a, ma = _run(cuda_lib, keys, g, 1e-3, [], t, entry="objects")
        b, mb = _run(cuda_lib, keys, g, 1e-3, [], t, entry="plain")
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)) and ma == mb
    cfg = Config(domain_bits=DOMAIN_BITS)
    sdf, grad = levelset.sphere(cfg, (0.52, 0.47, 0.5), 0.21)
    gsz = cfg.grid_size
    field = np.ascontiguousarray(np.concatenate([sdf[None], grad]).reshape(4, gsz, 4, gsz, 4, gsz, 4).transpose(1, 3, 5, 0, 2, 4, 6).reshape(-1)).astype(np.float32)
    t_field = torch.from_numpy(field).cuda()
    col = Collider()
    col.sdf = t_field.data_ptr()
    col.rot_mat[:] = [1, 0, 0, 0, 1, 0, 0, 0, 1]
    col.trans_vel[:] = [0.2, 0.0, 0.0]
    col.scale, col.type, col.friction = 1.0, 1, 0.3
    a, ma = _run(cuda_lib, keys, g, 1e-3, [], 0.37, col=col, entry="objects")
    b, mb = _run(cuda_lib, keys, g, 1e-3, [], 0.37, col=col, entry="collider")
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)) and ma == mb
    # with the collider and objects both present the collider resolves first: a sticky object after it decides alone where it hits
    obj = objects.box((0.3, 0.28, 0.33), (0.68, 0.61, 0.7), type="sticky")
    c, _ = _run(cuda_lib, keys, g, 1e-3, [obj], 0.37, col=col, entry="objects")
    d, _ = _run(cuda_lib, keys, g, 1e-3, [obj], 0.37, entry="objects")
    ref, _, _, info = ref64.grid_update(cfg, keys, g, 1e-3, None, np.float32(0.37), objects=[obj])
    near = info["near"]
    hit = (ref == 0).all(1) & (g[:, 0] > 0) & ~near
    assert hit.sum() > 1000
    assert np.array_equal(c[:, 1:][np.broadcast_to(hit[:, None], ref.shape)], d[:, 1:][np.broadcast_to(hit[:, None], ref.shape)])
    assert (c != d).any()


# ---- kernel level against the oracle, with and without the level-set collider --------------------------------------------------
def _sphere_field(cfg):
    sdf, grad = levelset.sphere(cfg, (0.42, 0.30, 0.40), 0.09)
    g = cfg.grid_size
    return np.ascontiguousarray(np.concatenate([sdf[None], grad]).reshape(4, g, 4, g, 4, g, 4).transpose(1, 3, 5, 0, 2, 4, 6).reshape(-1)).astype(np.float32)


def _collider_pair(field_ptr_engine, field_ptr_oracle, typ=1, friction=0.3, trans_vel=(0.2, 0.0, 0.0)):
    out = []
    for cls, ptr in ((Collider, field_ptr_engine), (cob.Collider, field_ptr_oracle)):
        c = cls()
        c.sdf = ptr
        c.rot_mat[:] = [1, 0, 0, 0, 1, 0, 0, 0, 1]
        c.trans_vel[:] = list(trans_vel)
        c.scale, c.type, c.friction = 1.0, typ, friction
        out.append(c)
    return out


OVERLAP = {
    # lattice-aligned and static: the nodes equidistant from two faces are exact ties in float32 (the lowest axis must win)
    "lattice_box": lambda: [objects.box((0.25, 0.25, 0.25), (0.5, 0.5, 0.5), type="slip", friction=0.0)],
    "two": lambda: [objects.box((0.3, 0.2, 0.3), (0.55, 0.34, 0.55), type="slip", friction=0.3, **MOTIONS["combined"]),
                    objects.sphere((0.45, 0.3, 0.45), 0.1, type="separate", friction=0.2, trans_vel=(0.1, 0.0, 0.0))],
    "three": lambda: [objects.plane((0.5, 0.3, 0.5), (0.1, 1.0, 0.0), type="sticky"),
                      objects.cylinder((0.4, 0.3, 0.4), 0.08, 0.1, type="slip", friction=0.0, omega=(0.0, 0.7, 0.0)),
                      objects.box((0.35, 0.25, 0.35), (0.5, 0.4, 0.5), type="separate", friction=0.3, rot=_rot(0.2, 0.1, 0.0))],
}


@pytest.mark.parametrize("t", [0.0, 0.37, 3.1])
@pytest.mark.parametrize("collider", [False, True], ids=["objects", "levelset+objects"])
@pytest.mark.parametrize("case", sorted(OVERLAP))
def test_kernel_matches_oracle(oracle, cuda_lib, grid, case, collider, t):
    """test_gpu_collider.test_kernel_matches_oracle's bounds: velocity per cell rel 1e-6 with an absolute floor of 1e-5 max|v|
    (rotating objects), max |v|^2 rel 1e-6."""
    torch = _torch()
    keys, g = grid
    cfg = Config(domain_bits=DOMAIN_BITS)
    ocfg = ob.make_config(domain_bits=DOMAIN_BITS)
    objs = OVERLAP[case]()
    field = _sphere_field(cfg)
    t_field = torch.from_numpy(field).cuda()
    ecol, ocol = _collider_pair(t_field.data_ptr(), field.ctypes.data)
    og = g.reshape(-1).copy()
    part = ob.Partition()
    part.active_keys = keys.ctypes.data
    omv = np.zeros(1, np.float32)
    arr = cob.unit_planes(objs)
    cob.lib().orc_update_grid_velocity_query_max_boundaries(C.byref(ocfg), len(keys), ob.ptr(og), part, 1e-3, C.byref(ocol) if collider else None, arr, len(objs),
                                                            np.float32(t), ob.ptr(omv))
    eg, emx = _run(cuda_lib, keys, g, 1e-3, objs, np.float32(t), col=ecol if collider else None)
    og = og.reshape(g.shape)
    scale = np.abs(og[:, 1:]).max()
    assert np.allclose(eg[:, 1:], og[:, 1:], rtol=1e-6, atol=1e-5 * scale), np.abs(eg[:, 1:] - og[:, 1:]).max() / scale
    assert emx == pytest.approx(float(omv[0]), rel=1e-6)
    changed = (og[:, 1:] != g[:, 1:] / np.where(g[:, 0] > 0, g[:, 0], 1)[:, None]).any(1) & (g[:, 0] > 0)
    assert changed.sum() > 100


def test_sphere_object_matches_levelset_collider_away_from_surface(cuda_lib, grid):
    """The response (collider_resolve) over its two queries on identical inputs: a sphere object and the
    level-set collider on levelset.sphere's field, same type, friction and motion, give the same velocities at every node a cell or
    more from the surface and off the sphere's centre (the trilinear gradient there is the exact normal up to float32 rounding)."""
    torch = _torch()
    keys, g = grid
    cfg = Config(domain_bits=DOMAIN_BITS)
    dx = cfg.dx
    centre, radius = (0.4375, 0.40625, 0.4375), 0.15   # on the lattice
    sdf, grad = levelset.sphere(cfg, centre, radius)
    gs = cfg.grid_size
    field = np.ascontiguousarray(np.concatenate([sdf[None], grad]).reshape(4, gs, 4, gs, 4, gs, 4).transpose(1, 3, 5, 0, 2, 4, 6).reshape(-1)).astype(np.float32)
    t_field = torch.from_numpy(field).cuda()
    nodes = keys[:, None, :] * 4 + np.stack(np.meshgrid(np.arange(4), np.arange(4), np.arange(4), indexing="ij"), -1).reshape(1, 64, 3)
    r = np.sqrt(((nodes * dx - np.asarray(centre)) ** 2).sum(-1))
    far = (np.abs(r - radius) > 1.5 * dx) & (r > 1.5 * dx)
    for typ in (0, 1, 2):
        ecol, _ = _collider_pair(t_field.data_ptr(), 0, typ=typ, friction=0.3, trans_vel=(0.0, 0.0, 0.0))
        a, _ = _run(cuda_lib, keys, g, 1e-3, [], 0.0, col=ecol, entry="collider")
        b, _ = _run(cuda_lib, keys, g, 1e-3, [objects.sphere(centre, radius, type=typ, friction=0.3)], 0.0)
        inside = far & (r < radius) & (g[:, 0] > 0)
        assert inside.sum() > 1000
        da = np.transpose(a[:, 1:], (0, 2, 1))[far]
        db = np.transpose(b[:, 1:], (0, 2, 1))[far]
        assert np.allclose(da, db, rtol=1e-5, atol=1e-5 * np.abs(da).max()), typ


# ---- step driver against the oracle -------------------------------------------------------------------------------------------
FLOOR = ((0.15, 0.15, 0.15), (0.85, 0.305, 0.85))


def _set_both(osim, esim, objs):
    osim.set_collision_objects(objs)
    esim.set_collision_objects(objs)


def _sticky_floor_dt_scene():
    return scenes.small_cube(v0=(1.0, -10.0, 0.5))


@pytest.mark.timeout(600)
@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
@pytest.mark.parametrize("typ", ["sticky", "slip", "separate"])
@pytest.mark.parametrize("material", [scenes.FIXED_COROTATED, scenes.J_FLUID, scenes.SAND, scenes.NACC])
def test_cube_on_analytic_floor_matches_oracle(oracle, cuda_lib, material, typ, use_graph):
    scene = scenes.small_cube(material=material, v0=(0.3, -1.5, 0.2))
    osim = ts.build_oracle(ob, scene, sim_class=cob.ColliderOracleSim)
    esim = scenes.build_engine(scene, use_graph=use_graph)
    _set_both(osim, esim, [objects.box(*FLOOR, type=typ, friction=0.3)])
    for k in range(4):
        osim.step(10)
        esim.step(10)
        tgc._compare_state(osim, esim, f"{typ} after {10 * (k + 1)} sub-steps", f_tol=2e-4 if material in (scenes.SAND, scenes.NACC) else 5e-5)
    assert esim.sim_time() == pytest.approx(osim.sim_time, rel=1e-6)
    esim.close()


@pytest.mark.timeout(600)
def test_fluid_in_five_planes_matches_oracle(oracle, cuda_lib):
    scene = scenes.small_cube(material=scenes.J_FLUID, lo=18, hi=34, v0=(0.8, -1.0, -0.6))
    osim = ts.build_oracle(ob, scene, sim_class=cob.ColliderOracleSim)
    esim = scenes.build_engine(scene)
    walls = [objects.plane((0.5, 0.27, 0.5), (0, 1, 0), type="slip", friction=0.0),
             objects.plane((0.27, 0.5, 0.5), (1, 0, 0), type="separate", friction=0.2),
             objects.plane((0.54, 0.5, 0.5), (-1, 0, 0), type="slip", friction=0.3),
             objects.plane((0.5, 0.5, 0.27), (0, 0, 1), type="sticky"),
             objects.plane((0.5, 0.5, 0.54), (0, 0, -1), type="separate", friction=0.0)]
    _set_both(osim, esim, walls)
    for k in range(4):
        osim.step(10)
        esim.step(10)
        tgc._compare_state(osim, esim, f"planes after {10 * (k + 1)} sub-steps")
    esim.close()


@pytest.mark.timeout(600)
def test_fluid_with_moving_cylinder_paddle_matches_oracle(oracle, cuda_lib):
    scene = scenes.small_cube(material=scenes.J_FLUID, lo=18, hi=34, v0=(0.0, 0.0, 0.0))
    osim = ts.build_oracle(ob, scene, sim_class=cob.ColliderOracleSim)
    esim = scenes.build_engine(scene)
    paddle = objects.cylinder((0.26, 0.4, 0.40), 0.04, 0.2, type="slip", friction=0.0, trans_vel=(1.5, 0.0, 0.0), omega=(0.0, 0.5, 0.0), trans=(0.26, 0.4, 0.4))
    _set_both(osim, esim, [paddle])
    for k in range(4):
        osim.step(10)
        esim.step(10)
        tgc._compare_state(osim, esim, f"paddle after {10 * (k + 1)} sub-steps")
    esim.close()


@pytest.mark.timeout(600)
@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
def test_levelset_collider_with_two_objects_matches_oracle(oracle, cuda_lib, use_graph):
    scene = scenes.small_cube(v0=(0.3, -1.5, 0.2))
    osim = ts.build_oracle(ob, scene, sim_class=cob.ColliderOracleSim)
    esim = scenes.build_engine(scene, use_graph=use_graph)
    p = tgc._params("slip", 0.3, "trans_vel")
    tgc._set_both(osim, esim, scene["domain_bits"], "sphere", p)
    objs = [objects.box(*FLOOR, type="sticky", trans_vel=(0.1, 0.0, 0.0)), objects.sphere((0.5, 0.38, 0.45), 0.06, type="separate", friction=0.3)]
    _set_both(osim, esim, objs)
    for k in range(4):
        osim.step(10)
        esim.step(10)
        tgc._compare_state(osim, esim, f"collider + objects after {10 * (k + 1)} sub-steps")
    esim.close()


@pytest.mark.timeout(600)
@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
def test_set_and_clear_between_substeps(oracle, cuda_lib, use_graph):
    scene = scenes.small_cube(v0=(0.3, -1.5, 0.2))
    osim = ts.build_oracle(ob, scene, sim_class=cob.ColliderOracleSim)
    esim = scenes.build_engine(scene, use_graph=use_graph)
    osim.step(10)
    esim.step(10)
    _set_both(osim, esim, [objects.box(*FLOOR, type="sticky", friction=0.3, trans_vel=(0.3, 0.5, -0.2))])
    osim.step(10)
    esim.step(10)
    tgc._compare_state(osim, esim, "objects set")
    osim.set_collision_objects([])
    esim.clear_collision_objects()
    osim.step(10)
    esim.step(10)
    tgc._compare_state(osim, esim, "objects cleared")
    _set_both(osim, esim, [objects.plane((0.5, 0.29, 0.5), (0.1, 1.0, 0.0), type="slip", friction=0.2), objects.box(*FLOOR, type="separate")])
    osim.step(10)
    esim.step(10)
    tgc._compare_state(osim, esim, "objects set again")
    esim.close()


@pytest.mark.timeout(600)
@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
def test_emission_with_objects_matches_oracle(oracle, cuda_lib, use_graph):
    """Particles added with objects set re-capture the sub-step graphs: the sub-steps after it still match the oracle, which is
    built with the same particles from the start and so needs the objects at the same times."""
    scene = scenes.small_cube(material=scenes.J_FLUID, v0=(0.0, -1.0, 0.0))
    extra = scene["models"][0]["pos"] + np.float32([0.0, 0.0, 0.25])
    esim = scenes.build_engine(scene, use_graph=use_graph)
    floor = [objects.box(*FLOOR, type="slip", friction=0.3, trans_vel=(0.2, 0.0, 0.0))]
    esim.set_collision_objects(floor)
    esim.add_particles(0, extra, (0.0, -1.0, 0.0))
    both = dict(scene, models=[dict(scene["models"][0], pos=np.concatenate([scene["models"][0]["pos"], extra]))])
    osim = ts.build_oracle(ob, both, sim_class=cob.ColliderOracleSim)
    osim.set_collision_objects(floor)
    for k in range(4):
        osim.step(10)
        esim.step(10)
        tgc._compare_state(osim, esim, f"emitted, after {10 * (k + 1)} sub-steps")
    esim.close()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("use_graph", [True, False], ids=["graph", "stream"])
def test_mgsp_two_ranks_analytic_sticky_floor_match_single_domain(oracle, cuda_lib, use_graph):
    """The max |v|^2 the ranks agree on comes from the objects instances of grid_max_boundary_kernel at set-up and of
    carry_grid_boundary_kernel after each sub-step: with a CFL-bound dt (fast cube, dt_default 1e-3) it drives dt, which must equal the single-domain oracle's (whose max
    is the one its grid update finds) and be bit-identical on both ranks."""
    from claymore_b200 import mgsp
    scene = _sticky_floor_dt_scene()
    dt_default = 1e-3
    osim = ts.build_oracle(ob, scene, dt=dt_default, sim_class=cob.ColliderOracleSim)
    # the floor rises at 6 m/s under the falling cube: a sticky object's velocity (2 trans_vel, 12 m/s) exceeds the cube's, so the
    # predicted max, and so dt, is wrong wherever a predictor leaves the objects out
    floor = [objects.box((0.15, 0.15, 0.15), (0.85, 0.33, 0.85), type="sticky", friction=0.3, trans_vel=(0.0, 6.0, 0.0)),
             objects.sphere((0.45, 0.6, 0.45), 0.05, type="slip", trans_vel=(0.5, 0.0, 0.0))]
    osim.set_collision_objects(floor)
    sims = []
    for r in range(2):
        sims.append(mgsp.build_rank_sim(mgsp.partition_scene(scene, r, 2), r, 2, dt_default, 4000, ts.apply_material, use_graph=use_graph))
        sims[-1].set_collision_objects(floor)
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
    bound = False
    for k in range(4):
        osim.step(5)
        run(lambda s: (s.step(5), s.sync()))
        sts = [s.stats() for s in sims]
        assert all(st.error == 0 for st in sts)
        assert np.float32(sts[0].dt).view(np.uint32) == np.float32(sts[1].dt).view(np.uint32), (k, sts[0].dt, sts[1].dt)
        assert sts[0].dt == pytest.approx(osim.dt, rel=1e-5), (k, sts[0].dt, osim.dt)
        bound |= osim.dt < dt_default * 0.99
        pos = np.concatenate([s.retrieve(0) for s in sims])
        opos = osim.retrieve(0)
        assert len(pos) == len(opos)
        ts.match_particles(opos, pos, tol=2e-6)
    assert bound, "the CFL condition must bind dt"
    for s in sims:
        s.close()


@pytest.mark.timeout(600)
def test_scene_boundaries_equal_api_calls_and_resume(oracle, cuda_lib, tmp_path):
    from claymore_b200 import scene
    doc = {"simulation": {"default_dt": 1e-4, "fps": 24, "frames": 2},
           "models": [{"constitutive": "jfluid", "file": "box", "offset": [0.35, 0.35, 0.35], "span": [0.2, 0.2, 0.2], "velocity": [0.2, -1.0, 0],
                       "rho": 1000, "volume": 1e-6, "bulk_modulus": 1e4, "gamma": 7.15, "viscosity": 0.0}],
           "boundaries": [{"shape": "box", "offset": [0.1, 0.1, 0.1], "span": [0.8, 0.25, 0.8], "type": "slip", "friction": 0.2},
                          {"shape": "cylinder", "offset": [0.3, 0.3, 0.3], "span": [0.06, 0.4, 0.06], "velocity": [0.5, 0, 0]}]}
    cfg = Config(domain_bits=6)
    a = scene.parse_scene(doc, config=cfg, max_blocks=4000)
    b = scene.parse_scene(dict(doc, boundaries=[]), config=cfg, max_blocks=4000)
    b.set_collision_objects([objects.box((0.1, 0.1, 0.1), (0.9, 0.35, 0.9), type="slip", friction=0.2),
                             objects.cylinder((0.33, 0.5, 0.33), 0.03, 0.2, trans_vel=(0.5, 0, 0))])
    for s in (a, b):
        s.initial_setup()
        s.step(30)
    tgc._same_state(a, b)
    # a checkpoint of the scene resumes with its boundaries: test_gpu_checkpoint's continuation bounds against the uninterrupted run
    path = str(tmp_path / "ck.bin")
    a.save_checkpoint(path)
    c = scene.parse_scene(doc, config=cfg, max_blocks=4000, resume=path)
    a.step(20)
    c.step(20)
    tgc._same_state(a, c)
    for s in (a, b, c):
        s.close()
