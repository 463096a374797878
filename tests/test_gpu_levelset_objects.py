"""GPU tests of the level-set collision objects (CB200_SHAPE_LEVELSET, DESIGN.md section 2.11).

Prepare: cb200_levelset_prepare against numpy's float32 central differences bit for bit.  Kernel: the grid update with level-set
objects against the float64 reference (ref64 with ref64_levelset's query) per node: |v - ref| within the larger of
test_gpu_objects' 1e-5 (1 + |v_ref|) and COLLIDER_VEL_KAPPA 2^-24 E (E carries the normal's sensitivity to the rounding of the
query point, large on a coarse lattice), flagged nodes at most 2 %; list order; the dense collider's field as a level-set object bit
for bit outside the wall band; a level set of a sphere against the analytic sphere.  Step driver (g2p2g's float atomics make two
runs differ in the last bits, so runs are compared particle by particle within STEP_TOL): the same field as object and as dense
collider, graph and stream mode with a moving obstacle and registration and clearing between sub-steps.  Sinks: removal by a
level-set region against ref64_levelset's hit set.  Scene: .sdf boundaries and sinks against the same API calls."""
import ctypes as C
import json

import numpy as np
import pytest

import ref64
import ref64_cases as S
import ref64_levelset as RL
import sdf_ref
from claymore_b200 import _capi, objects, samplers, scene, sdf
from claymore_b200._capi import CB200Error, CollisionObject, Config, LevelSetLattice, Partition, SdfHeader
from claymore_b200.simulator import GmpmSimulator
from ref64_checks import COLLIDER_VEL_KAPPA
from scenes import match_particles
from test_levelset_objects_cpu import LATTICES, level_set

pytestmark = pytest.mark.gpu
DOMAIN_BITS = 6
DX = 1.0 / (1 << DOMAIN_BITS)
STEP_TOL = 1e-4   # positions (m) and every other channel (relative to its largest value) of two runs of the same scene


def _torch():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch


def _rot(ax, ay, az):
    cx, sx, cy, sy, cz, sz = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay), np.cos(az), np.sin(az)
    return np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]]) @ np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])


MOTIONS = {"static": {}, "combined": dict(rot=_rot(0.3, -0.2, 0.5), trans=(0.5, 0.47, 0.5), trans_vel=(0.04, -0.03, 0.02), omega=(0.3, -0.2, 0.5),
                                          scale=1.15, dsdt=0.2)}
# each level set fitted into a box around the grid's middle: (offset, span)
PLACEMENT = {"sphere": ((0.3, 0.28, 0.3), (0.4, 0.4, 0.4)), "torus": ((0.25, 0.35, 0.25), (0.5, 0.5, 0.5)),
             "box": ((0.3, 0.25, 0.3), (0.4, 0.45, 0.4)), "plate": ((0.25, 0.3, 0.25), (0.5, 0.5, 0.5)),
             "dragonish": ((0.4, 0.3, 0.2), (0.6, 0.6, 0.6))}


def _lattice_dev(lat):
    torch = _torch()
    return torch.from_numpy(np.ascontiguousarray(lat, np.float32).reshape(-1)).cuda()


def _prepare(n, phi):
    torch = _torch()
    d_phi = torch.from_numpy(np.ascontiguousarray(phi, np.float32).reshape(-1)).cuda()
    out = torch.empty(4 * d_phi.numel(), dtype=torch.float32, device="cuda")
    h = SdfHeader(n[0], n[1], n[2], (C.c_float * 3)(0, 0, 0), 0.1)
    assert _capi.lib().cb200_levelset_prepare(C.byref(h), C.c_void_p(d_phi.data_ptr()), C.c_void_p(out.data_ptr()), None) == 0
    torch.cuda.synchronize()
    return out.cpu().numpy().reshape(n[2], n[1], n[0], 4)


@pytest.fixture(scope="module")
def grid():
    """every block of [2, 14)^3 on a 64^3 grid, masses log-uniform in [1e-3, 1] with some empty nodes, velocities N(0, 2)"""
    rng = np.random.default_rng(11)
    r = np.arange(2, 14)
    keys = np.stack(np.meshgrid(r, r, r, indexing="ij"), -1).reshape(-1, 3).astype(np.int32)
    nb = len(keys)
    g = np.zeros((nb, 4, 64), np.float32)
    m = np.exp(rng.uniform(np.log(1e-3), 0.0, (nb, 64))).astype(np.float32)
    m[rng.random((nb, 64)) < 0.05] = 0.0
    g[:, 0] = m
    g[:, 1:] = (rng.normal(0, 2.0, (nb, 3, 64)) * m[:, None]).astype(np.float32)
    return keys, g


def _run(keys, g, dt, objs, t, lattices=(), col=None, entry="levelsets"):
    """the kernel-level grid update; lattices: float32[nk, nj, ni, 4] arrays, registry order"""
    torch = _torch()
    lib = _capi.lib()
    t_g = torch.from_numpy(g.reshape(-1).copy()).cuda()
    t_k = torch.from_numpy(keys.reshape(-1).copy()).cuda()
    t_mv = torch.zeros(1, dtype=torch.float32, device="cuda")
    part = Partition()
    part.active_keys = t_k.data_ptr()
    cfg = Config(domain_bits=DOMAIN_BITS)
    arr = (CollisionObject * max(len(objs), 1))(*objs)
    G, MV = C.c_void_p(t_g.data_ptr()), C.c_void_p(t_mv.data_ptr())
    if entry == "collider":
        e = lib.cb200_update_grid_velocity_query_max_collider(C.byref(cfg), len(keys), G, part, dt, C.byref(col), t, MV, None)
    else:
        devs = [_lattice_dev(l) for l in lattices]
        views = (LevelSetLattice * max(len(devs), 1))(*[LevelSetLattice(d.data_ptr(), l.shape[2], l.shape[1], l.shape[0]) for d, l in zip(devs, lattices)])
        e = lib.cb200_update_grid_velocity_query_max_levelsets(C.byref(cfg), len(keys), G, part, dt, C.byref(col) if col is not None else None, arr,
                                                              len(objs), views, len(devs), t, MV, None)
    assert e == 0
    torch.cuda.synchronize()
    return t_g.cpu().numpy().reshape(g.shape), float(t_mv.item())


def _obj(name, index=0, **kw):
    ls = level_set(name)
    o = objects.levelset(ls, *PLACEMENT[name], **kw)
    o.b[1] = float(index)
    return o, RL.lattice(ls.n, ls.phi)


# ---- prepare --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(LATTICES) + ["two_wide"])
def test_prepare_equals_numpy_bit_for_bit(name):
    if name == "two_wide":
        n, _, phi = sdf_ref.sphere((2, 7, 5), 0.3, (0.1, 0.9, 0.6), 0.5)
    else:
        n, _, phi = LATTICES[name]()
    got, want = _prepare(n, phi), RL.lattice(n, phi)
    assert got.view(np.uint32).tobytes() == want.view(np.uint32).tobytes()


# ---- kernel against ref64 ---------------------------------------------------------------------------------------------------------
def _check(grid, objs, lattices, t, dt=1e-3, col=None):
    keys, g = grid
    eg, emx = _run(keys, g, dt, objs, t, lattices, col)
    with RL.registered(lattices):
        ref, vmag, _, info = ref64.grid_update(Config(domain_bits=DOMAIN_BITS), keys, g, dt, None, t, objects=objs)
    near = info["near"]
    has = g[:, 0] >= np.finfo(np.float32).tiny
    ok = has & ~near
    err = np.abs(eg[:, 1:] - ref)
    bound = np.maximum(1e-5 * (1 + np.abs(ref).max(1))[:, None], COLLIDER_VEL_KAPPA * ref64.EPS32 * vmag)
    err = (err / bound).max(1)
    bound = np.ones_like(err)
    assert (err[ok] <= bound[ok]).all(), float((err[ok] / bound[ok]).max())
    assert near[has].mean() <= 0.02, near[has].mean()
    vsq = (eg[:, 1:].astype(np.float64) ** 2).sum(1)[has]
    assert emx == pytest.approx(vsq.max(), rel=1e-6)
    hit = np.zeros_like(ok)
    for st in info["stages"]:   # nodes some object of the list hits, away from every margin
        hit |= st["hit"].astype(bool)
    return ok.sum(), (hit & ok).sum()


@pytest.mark.parametrize("t", [0.0, 0.37, 3.1])
@pytest.mark.parametrize("motion", sorted(MOTIONS))
@pytest.mark.parametrize("friction", [0.0, 0.3])
@pytest.mark.parametrize("typ", ["sticky", "slip", "separate"])
@pytest.mark.parametrize("name", list(LATTICES))
def test_kernel_matches_reference(grid, name, typ, friction, motion, t):
    o, lat = _obj(name, type=typ, friction=friction, **MOTIONS[motion])
    _, hit = _check(grid, [o], [lat], np.float32(t))
    assert hit > 100, "the object must act on the grid"


@pytest.mark.parametrize("t", [0.0, 3.1])
def test_levelset_between_analytic_objects_in_list_order(grid, t):
    ls_obj, lat = _obj("sphere", index=0, type="slip", friction=0.3, **MOTIONS["combined"])
    objs = [objects.box((0.35, 0.3, 0.35), (0.7, 0.6, 0.65), type="sticky", trans_vel=(0.1, 0.0, 0.0)), ls_obj,
            objects.cylinder((0.45, 0.5, 0.5), 0.15, 0.2, type="separate", friction=0.0, omega=(0.0, 0.7, 0.0))]
    _check(grid, objs, [lat], np.float32(t))
    _check(grid, objs[::-1], [lat], np.float32(t))
    keys, g = grid
    a, _ = _run(keys, g, 1e-3, objs, np.float32(t), [lat])
    b, _ = _run(keys, g, 1e-3, objs[::-1], np.float32(t), [lat])
    assert (a != b).any(), "overlapping objects depend on the list order"


def test_two_levelsets_index_their_own_lattice(grid):
    a, la = _obj("torus", index=1, type="slip", friction=0.3)
    b, lb = _obj("box", index=0, type="separate", friction=0.0)
    _check(grid, [a, b], [lb, la], np.float32(0.0))


# ---- cross-checks ------------------------------------------------------------------------------------------------------------------
def _interior_field(boundary=2):
    """the dense collider's (sdf, grad) with grad replaced, inside the wall band, by the lattice the interior nodes' phi prepares to:
    (sdf, grad, lattice, first interior node)"""
    sdf_d, _ = S.make_field(DOMAIN_BITS, ("sphere", (0.52, 0.47, 0.5), 0.21))
    N = sdf_d.shape[0]
    lo, hi = 4 * boundary, N - 4 * boundary
    sub = sdf_d[lo:hi, lo:hi, lo:hi]
    m = hi - lo
    lat = RL.lattice((m, m, m), np.transpose(sub, (2, 1, 0)))                 # [k, j, i] order: i = x
    grad = np.zeros((3, N, N, N), np.float32)
    for d in range(3):
        grad[d, lo:hi, lo:hi, lo:hi] = np.transpose(lat[..., 1 + d], (2, 1, 0))
    return sdf_d, grad, lat, lo


@pytest.mark.parametrize("typ", ["sticky", "slip", "separate"])
def test_lattice_on_the_grid_nodes_equals_the_dense_collider_bit_for_bit(grid, typ):
    """a = the first interior node, c = dx: q is integral at every node, so the interpolation is exact and the object must give
    what the dense collider gives, outside the wall band (where the collider reports no hit)"""
    from test_ref64_collider_cpu import block_field
    torch = _torch()
    keys, g = grid
    sdf_d, grad, lat, lo = _interior_field()
    field = torch.from_numpy(block_field(DOMAIN_BITS, sdf_d, grad)).cuda()
    col = S.collider_struct(_capi.Collider(), dict(type={"sticky": 0, "slip": 1, "separate": 2}[typ], friction=0.3))
    col.sdf = field.data_ptr()
    o = objects.box((0, 0, 0), (1, 1, 1), type=typ, friction=0.3)
    o.shape = _capi.SHAPE_LEVELSET
    o.a[:] = (lo * DX,) * 3
    o.b[:] = (DX, 0.0, 0.0)
    a, _ = _run(keys, g, 1e-3, [], np.float32(0.0), col=col, entry="collider")
    b, _ = _run(keys, g, 1e-3, [o], np.float32(0.0), [lat])
    assert a.view(np.uint32).tobytes() == b.view(np.uint32).tobytes()


def test_zero_phi_is_solid(grid):
    """a plane level set phi = j - 4 on nodes c = dx apart, aligned with the grid: the node layer where phi is exactly 0 is solid
    (phi <= 0, as the dense collider and the other shapes), the layer above is not"""
    keys, g = grid
    n = (12, 12, 12)
    phi = np.broadcast_to((np.arange(n[1], dtype=np.float32) - 4.0)[None, :, None], (n[2], n[1], n[0]))
    o = objects.box((0, 0, 0), (1, 1, 1), type="sticky")
    o.shape = _capi.SHAPE_LEVELSET
    o.a[:] = (20 * DX,) * 3
    o.b[:] = (DX, 0.0, 0.0)
    a, _ = _run(keys, g, 1e-3, [o], np.float32(0.0), [RL.lattice(n, phi)])
    has = g[:, 0] >= np.finfo(np.float32).tiny
    node = keys[:, None, :] * 4 + ref64._CELLS[None]
    inside = np.all((node >= 20) & (node <= 31), axis=2)
    hit = (a[:, 1:] == 0).all(1)
    for j, solid in ((24, True), (25, False), (20, True)):
        on = has & inside & (node[..., 1] == j)
        assert on.sum() > 20 and (hit[on] == solid).all(), (j, solid)


def test_levelset_sphere_hits_the_analytic_sphere(grid):
    """sticky and static: a hit node's velocity becomes exactly 0; away from the surface (0.3 c), the hit sets agree"""
    keys, g = grid
    n, h, phi = sdf_ref.sphere((33, 33, 33), 0.05, (0.8, 0.8, 0.8), 0.6)
    ls = sdf.parse(sdf_ref.text(n, h, phi))
    offset, span = (0.3, 0.3, 0.3), (0.4, 0.4, 0.4)
    c, lo, _ = sdf.node_box(ls, offset, span)
    centre, r = np.array(lo) + 0.8 / 0.05 * c, 0.6 / 0.05 * c
    a, _ = _run(keys, g, 1e-3, [objects.levelset(ls, offset, span, type="sticky")], np.float32(0.0), [RL.lattice(n, phi)])
    b, _ = _run(keys, g, 1e-3, [objects.sphere(centre, r, type="sticky")], np.float32(0.0))
    has = g[:, 0] >= np.finfo(np.float32).tiny
    nodes = (keys[:, None, :] * 4 + ref64._CELLS[None]).astype(np.float64) * DX
    dist = np.linalg.norm(nodes - centre, axis=2)
    far = has & (np.abs(dist - r) > 0.3 * c)
    hit_a, hit_b = (a[:, 1:] == 0).all(1), (b[:, 1:] == 0).all(1)
    assert hit_b[far].sum() > 1000
    assert np.array_equal(hit_a[far], hit_b[far])


# ---- step driver ------------------------------------------------------------------------------------------------------------------
def _sim(use_graph=True, material=_capi.SAND, v0=(0.3, -1.0, 0.2)):
    s = GmpmSimulator(config=Config(domain_bits=DOMAIN_BITS), dt=1e-3, max_blocks=4000, use_graph=use_graph)
    s.init_model(material, samplers.uniform_box(DX, (24, 30, 24), (36, 38, 34)), v0)
    s.initial_setup()
    return s


def _same_run(a, b):
    """two simulators of the same scene: the same clock and error bits, and the same particles within STEP_TOL"""
    assert a.sim_time() == b.sim_time() and a.stats().error == b.stats().error
    for m in range(len(a.materials)):
        sa, sb = a.particle_state(m), b.particle_state(m)
        assert len(sa) == len(sb)
        idx = match_particles(sa, sb, STEP_TOL)
        assert np.abs(sb[idx][:, 3:] - sa[:, 3:]).max(initial=0.0) <= STEP_TOL * max(1.0, np.abs(sa[:, 3:]).max(initial=0.0))


def test_step_driver_lattice_on_nodes_equals_dense_collider():
    sdf_d, grad, lat, lo = _interior_field()
    a, b = _sim(), _sim()
    a.set_collider(sdf_d, grad, type="slip", friction=0.3)
    m = lat.shape[0]
    ls = sdf.LevelSet(SdfHeader(m, m, m, (C.c_float * 3)(0, 0, 0), 1.0), np.ascontiguousarray(lat[..., 0].reshape(-1)))
    idx = b.add_collision_levelset(ls)
    o = objects.box((0, 0, 0), (1, 1, 1), type="slip", friction=0.3)
    o.shape = _capi.SHAPE_LEVELSET
    o.a[:] = (lo * DX,) * 3
    o.b[:] = (DX, float(idx), 0.0)
    b.set_collision_objects([o])
    for _ in range(4):
        a.step(10)
        b.step(10)
        _same_run(a, b)
    assert a.stats().error == 0
    a.close(), b.close()


def _dragon_obstacle(**kw):
    ls = level_set("dragonish")
    return objects.levelset(ls, (0.3, 0.25, 0.2), (0.5, 0.5, 0.5), type="slip", friction=0.2, trans=(0.5, 0.4, 0.5), trans_vel=(0.0, 0.05, 0.0),
                            omega=(0.0, 0.6, 0.0), **kw)


def test_graph_and_stream_agree_with_moving_obstacle_and_changes_between_substeps():
    floor_ls = level_set("box")
    floor = objects.levelset(floor_ls, (0.1, 0.1, 0.1), (0.8, 0.3, 0.8), type="sticky")
    runs = []
    for use_graph in (True, False):
        s = _sim(use_graph, material=_capi.FIXED_COROTATED)
        s.set_collision_objects([floor, _dragon_obstacle()])
        s.step(10)
        s.set_collision_objects([_dragon_obstacle(), objects.plane((0.5, 0.15, 0.5), (0, 1, 0))])   # a new level set, reordered
        s.step(10)
        with pytest.raises(CB200Error):
            s.clear_collision_levelsets()                                  # still referenced
        s.set_collision_objects([objects.plane((0.5, 0.15, 0.5), (0, 1, 0))])
        s.clear_collision_levelsets()
        s.step(10)
        s.set_collision_objects([floor])                                   # registered again after the clear
        s.step(10)
        assert s.stats().error == 0
        runs.append(s)
    _same_run(*runs)
    for s in runs:
        s.close()


def test_registry_rejections():
    s = _sim()
    ls = level_set("plate")
    for _ in range(_capi.MAX_COLLISION_LEVELSETS):
        s.add_collision_levelset(sdf.parse(sdf_ref.text(ls.n, ls.h, ls.phi)))
    with pytest.raises(CB200Error):
        s.add_collision_levelset(ls)                                       # full
    o = objects.levelset(ls, (0.2, 0.2, 0.2), (0.5, 0.5, 0.5))
    del o.levelset
    o.b[1] = 16.0
    with pytest.raises(ValueError):
        s.set_collision_objects([o])
    assert s.L.cb200_sim_set_collision_objects(s.h, (CollisionObject * 1)(o), 1) == 1
    s.clear_collision_levelsets()
    o.b[1] = 0.0
    assert s.L.cb200_sim_set_collision_objects(s.h, (CollisionObject * 1)(o), 1) == 1   # the registry is empty again
    s.close()


# ---- sinks --------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("outside", [False, True])
@pytest.mark.parametrize("motion", ["static", "moving"])
def test_sink_removes_refs_set(outside, motion):
    s = _sim()
    s.step(3)
    kw = {} if motion == "static" else dict(trans=(0.5, 0.5, 0.5), trans_vel=(0.1, 0.0, -0.05), omega=(0.2, 0.5, 0.0))
    ls = level_set("torus")
    o = objects.levelset(ls, (0.3, 0.35, 0.3), (0.4, 0.4, 0.4), **kw)
    before = s.particle_state(0)
    t = s.sim_time()
    hit, near = RL.hits(o, RL.lattice(ls.n, ls.phi), np.float32(t), before[:, :3])
    gone = hit != outside
    removed = s.remove_particles([o], outside=outside)
    after = s.particle_state(0)
    assert removed[0] == len(before) - len(after)
    kept = {r.tobytes() for r in after}
    survived = np.array([r.tobytes() in kept for r in before])
    assert np.array_equal(~survived[~near], gone[~near])
    assert 0 < gone.sum() < len(before)
    s.step(2)
    assert s.stats().error == 0
    s.close()


def test_lattice_aligned_box_sink_selects_exactly():
    """a box level set on a lattice whose nodes are dx apart, aligned with the particles' own lattice: the float32 set is exact"""
    s = _sim()
    n = (9, 9, 9)
    phi = sdf_ref.box(n, 1.0, (2.0, 2.0, 2.0), (6.0, 6.0, 6.0))[2]
    ls = sdf.parse(sdf_ref.text(n, 1.0, phi))
    o = objects.levelset(ls, (26 * DX, 30 * DX, 26 * DX), (8 * DX,) * 3)
    before = s.particle_state(0)
    p = before[:, :3].astype(np.float64)
    lo, hi = np.array([28, 32, 28]) * DX, np.array([32, 36, 32]) * DX
    want = np.all((p >= lo) & (p <= hi), 1)
    removed = s.remove_particles([o])
    assert removed[0] == want.sum() > 0
    kept = {r.tobytes() for r in s.particle_state(0)}
    assert all((r.tobytes() in kept) != w for r, w in zip(before, want))
    s.close()


# ---- scene -------------------------------------------------------------------------------------------------------------------------
def test_scene_equals_api_calls(tmp_path):
    ls, box = level_set("dragonish"), level_set("box")
    (tmp_path / "dragon.sdf").write_bytes(sdf_ref.text(ls.n, ls.h, ls.phi))
    (tmp_path / "box.sdf").write_bytes(sdf_ref.text(box.n, box.h, box.phi))
    doc = {"simulation": {"frames": 3, "fps": 60, "default_dt": 1e-3},
           "models": [{"constitutive": "fixed_corotated", "file": "box", "offset": [0.375, 0.5, 0.375], "span": [0.1875, 0.125, 0.1875],
                       "velocity": [0, -1, 0], "rho": 1000, "volume": 1.0 / 64 ** 3 / 8, "youngs_modulus": 1e4, "poisson_ratio": 0.3}],
           "boundaries": [{"shape": "levelset", "file": "dragon.sdf", "offset": [0.3, 0.2, 0.2], "span": [0.5, 0.5, 0.5], "type": "slip",
                           "friction": 0.2, "omega": [0, 0.5, 0]}],
           "sinks": [{"shape": "levelset", "file": "box.sdf", "offset": [0.35, 0.45, 0.35], "span": [0.3, 0.3, 0.3], "start": 2}]}
    path = tmp_path / "scene.json"
    path.write_text(json.dumps(doc))
    a = scene.parse_scene(str(path), config=Config(domain_bits=DOMAIN_BITS), max_blocks=4000)
    a.main_loop()
    b = GmpmSimulator(dt=1e-3, fps=60, frames=3, config=Config(domain_bits=DOMAIN_BITS), max_blocks=4000)
    m = doc["models"][0]
    b.init_model(_capi.FIXED_COROTATED, scene._positions(m, b.cfg, str(tmp_path)), m["velocity"])
    b.update_fr_parameters(m["rho"], m["volume"], m["youngs_modulus"], m["poisson_ratio"], model=0)
    ls2 = sdf.read(str(tmp_path / "dragon.sdf"))
    b.set_collision_objects([objects.levelset(ls2, (0.3, 0.2, 0.2), (0.5, 0.5, 0.5), type="slip", friction=0.2, omega=(0, 0.5, 0))])
    sink = objects.levelset(sdf.read(str(tmp_path / "box.sdf")), (0.35, 0.45, 0.35), (0.3, 0.3, 0.3))
    b.emitters = [lambda s, f: s.remove_particles([sink]) if f >= 2 else None]
    b.main_loop()
    assert a.stats().error == 0 and b.stats().error == 0
    assert a.sim_time() >= 3 / 60 - 1e-3, "every frame must have run"
    assert len(a._levelsets) == 2 and len(b._levelsets) == 2
    _same_run(a, b)
    a.close(), b.close()


def test_scene_resume_equals_uninterrupted_run(tmp_path):
    """level sets are not in a checkpoint: a resumed scene registers its "boundaries" and "sinks" level sets again before the
    restore, and frames 4-6 (with the sink acting at 4 and 6) then equal the uninterrupted run within test_gpu_checkpoint's
    continuation bounds (a continuation differs only by the order of P2G's floating-point sums)"""
    import test_gpu_collider as tgc
    ls, box = level_set("dragonish"), level_set("box")
    (tmp_path / "dragon.sdf").write_bytes(sdf_ref.text(ls.n, ls.h, ls.phi))
    (tmp_path / "box.sdf").write_bytes(sdf_ref.text(box.n, box.h, box.phi))
    doc = {"simulation": {"frames": 6, "fps": 120, "default_dt": 1e-3},
           "models": [{"constitutive": "fixed_corotated", "file": "box", "offset": [0.375, 0.5, 0.375], "span": [0.1875, 0.125, 0.1875],
                       "velocity": [0, -1, 0], "rho": 1000, "volume": 1.0 / 64 ** 3 / 8, "youngs_modulus": 1e4, "poisson_ratio": 0.3}],
           "boundaries": [{"shape": "levelset", "file": "dragon.sdf", "offset": [0.42, 0.42, 0.25], "span": [0.5, 0.5, 0.5], "type": "slip",
                           "friction": 0.2, "omega": [0, 0.5, 0], "velocity": [0, 0.1, 0]}],
           "sinks": [{"shape": "levelset", "file": "box.sdf", "offset": [0.35, 0.45, 0.35], "span": [0.3, 0.3, 0.3], "start": 2, "every": 2}]}
    path = tmp_path / "scene.json"
    path.write_text(json.dumps(doc))
    cfg = Config(domain_bits=DOMAIN_BITS)
    ck = str(tmp_path / "f3.ckpt")
    a = scene.parse_scene(str(path), config=cfg, max_blocks=4000)
    n3 = {}

    def on_frame(s, f):
        if f == 3:
            s.save_checkpoint(ck)
            n3["count"] = s.counts[0]
    a.main_loop(on_frame=on_frame)
    assert a.stats().error == 0 and "count" in n3
    b = scene.parse_scene(str(path), config=cfg, max_blocks=4000, resume=ck)
    assert len(b._levelsets) == 1   # the boundary's, set before the restore; the sink registers its own when it first acts
    b.main_loop()
    assert b.stats().error == 0 and len(b._levelsets) == 2
    assert a.counts == b.counts
    tgc._same_state(a, b)
    a.close(), b.close()
