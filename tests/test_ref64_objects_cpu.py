"""The analytic collision objects against the float64 reference (ref64.object_chain), per node, per sub-step and in the dt.

Kernel level: orc_update_grid_velocity_query_max_boundaries on synthetic grids (blocks around each object's surface and centre,
masses log-uniform from 1e-12 to 1 with zero and subnormal nodes, velocities N(0, 2) m/s) over 4 shapes x 3 types x friction
{0, 0.3, -0.2} x {static, combined motion} x t {0, 0.37, 3.1} x boundary {2, 0}, plus the 16-object list and the level-set
collider with two objects.  Per node: |v - ref64| <= COLLIDER_VEL_KAPPA 2^-24 E, nodes near a discontinuity (ref64's margin)
left out and counted; the max within COLLIDER_MAX_REL of [mx_lo, mx_hi].  Per sub-step: the oracle with the objects through
OBJECT_CASES with COLLIDER_KAPPA.  The kappa values are the collider's (ref64_checks, test_ref64_collider_cpu): the oracle's worst ratios over this matrix
stay under them (printed per entry).  The GPU tests (test_gpu_objects_ref64.py) hold the engine to the same values.
"""
import ctypes as C

import numpy as np
import pytest

import ref64
import ref64_cases as S
from ref64_checks import MAX_NEAR_NODES, oracle_substep_check, ref_models
from test_ref64_collider_cpu import FIELDS, FRICTIONS, MOTIONS, TIMES, TYPES, block_field, check_collider_update, collider_of

DOMAIN_BITS = 6
SHAPES = {
    # off the lattice (no node within rounding of the plane), its normal stored as given: only the engine's normalisation
    # makes it a unit vector
    "plane": ("raw_plane", ((0.5, 0.4537, 0.5), (0.31, 1.0, -0.23))),
    "box": ("box", ((0.3, 0.28, 0.33), (0.68, 0.61, 0.7))),
    "sphere": ("sphere", ((0.5, 0.5, 0.5), 0.21)),                  # centred on a node: an exact zero normal when static
    # axis through nodes, r = 8 dx, h = 12 dx: zero normals on the side, and static exact cap / side ties where |d1| = rho + 4 dx
    "cylinder": ("cylinder", ((0.5, 0.5, 0.5), 0.125, 0.1875)),
}
ENTRIES = list(SHAPES) + ["sixteen", "levelset_objects"]
KERNEL_MATRIX = [(e, b, m) for e in ENTRIES for b in (2, 0) for m in MOTIONS]


def _motion(motion):
    """test_ref64_collider_cpu's motion as claymore_b200.objects keywords"""
    kw = dict(MOTIONS[motion])
    if "rot_mat" in kw:
        kw["rot"] = np.asarray(kw.pop("rot_mat"), np.float64).reshape(3, 3)
    return kw


make = S.make_object


def sixteen(k, motion):
    """16 objects, types and frictions rotated by k: five planes bounding the grid's middle and eleven small boxes and spheres."""
    kw = _motion(motion)
    tf = lambda i: dict(type=TYPES[(i + k) % 3], friction=FRICTIONS[(i + k) % 3])   # noqa: E731
    objs = [make("plane", ((0.5, 0.3, 0.5), (0.05, 1.0, 0.0)), **tf(0), **kw), make("plane", ((0.3, 0.5, 0.5), (1.0, 0.0, 0.1)), **tf(1), **kw),
            make("plane", ((0.7, 0.5, 0.5), (-1.0, 0.1, 0.0)), **tf(2), **kw), make("plane", ((0.5, 0.5, 0.3), (0.0, 0.0, 1.0)), **tf(3), **kw),
            make("plane", ((0.5, 0.5, 0.7), (0.1, 0.0, -1.0)), **tf(4), **kw)]
    for i in range(11):
        c = (0.36 + 0.027 * i, 0.4 + 0.03 * (i % 4), 0.35 + 0.028 * ((3 * i) % 11))
        if i % 2:
            objs.append(make("sphere", (c, 0.04), **tf(5 + i), **kw))
        else:
            objs.append(make("box", (tuple(x - 0.03 for x in c), tuple(x + 0.035 for x in c)), **tf(5 + i), **kw))
    return objs


def entry_runs(entry, motion):
    """(label, collider spec or None, objects) of one matrix entry and motion: every type and friction of a shape, three
    rotations of the 16-object list, three type choices of the level-set sphere with a box and a cylinder after it."""
    if entry in SHAPES:
        shape, args = SHAPES[entry]
        for typ in TYPES:
            for fr in FRICTIONS:
                yield f"type {typ} friction {fr}", None, [make(shape, args, type=typ, friction=fr, **_motion(motion))]
    elif entry == "sixteen":
        for k in range(3):
            yield f"rotation {k}", None, sixteen(k, motion)
    else:
        for k in range(3):
            spec = S.collider_spec(collider_of(TYPES[k], FRICTIONS[k], motion, "sphere"))
            yield f"collider type {TYPES[k]}", spec, [make("box", ((0.45, 0.3, 0.4), (0.6, 0.5, 0.62)), type=TYPES[(k + 1) % 3], friction=0.3, **_motion(motion)),
                                                      make("cylinder", ((0.5, 0.45, 0.5), 0.1, 0.12), type=TYPES[(k + 2) % 3], friction=-0.2, **_motion(motion))]


def kernel_config(ob, boundary):
    return ob.make_config(domain_bits=DOMAIN_BITS, boundary=boundary)


def _phi(o, x):
    """float64 signed distance (or a function with the same zero set) of object o (ref64.object_params) at points x[n, 3]"""
    a, b = o["a"], o["b"]
    if o["shape"] == ref64.PLANE:
        return (x - a) @ b
    if o["shape"] == ref64.BOX:
        return np.maximum(a - x, x - b).max(1)
    d = x - a
    if o["shape"] == ref64.SPHERE:
        return np.sqrt((d ** 2).sum(1)) - b[0]
    return np.maximum(np.sqrt(d[:, 0] ** 2 + d[:, 2] ** 2) - b[0], np.abs(d[:, 1]) - b[1])


def synthetic_grid(cfg, objs, spec, t, seed):
    """(keys int32, grid float32) as test_ref64_collider_cpu.synthetic_grid: up to 48 blocks with nodes within 2 dx of an
    object's surface, the blocks holding the spheres' and cylinders' centres, 4 blocks at the top face, 4 at the low x face
    and 4 anywhere."""
    rng = np.random.default_rng(seed)
    G = 1 << (cfg.domain_bits - 2)
    N, dx = 4 * G, 1.0 / (1 << cfg.domain_bits)
    nodes = np.stack(np.meshgrid(*[np.arange(N)] * 3, indexing="ij"), -1).reshape(-1, 3)
    near = np.zeros(len(nodes), bool)
    centres = []
    for o in objs:
        p = ref64.object_params(o)
        x = ref64.material_point(cfg, p, t, nodes)["x"][0]
        near |= np.abs(_phi(p, x)) < 2 * dx
        if p["shape"] in (ref64.SPHERE, ref64.CYLINDER):
            centres.append(nodes[np.argmin(((x - p["a"]) ** 2).sum(1))] >> 2)
        if p["shape"] == ref64.CYLINDER:   # the rim, where the cap / side switch lies (static: its exact ties at d2 = 0)
            for sx in (-1, 1):
                for sy in (-1, 1):
                    q = p["a"] + np.array([sx * (p["b"][0] - 2 * dx), sy * (p["b"][1] - 2 * dx), 0.0])
                    centres.append(nodes[np.argmin(((x - q) ** 2).sum(1))] >> 2)
    if spec is not None:
        sdf, _ = S.make_field(cfg.domain_bits, FIELDS["sphere"])
        x = ref64.material_point(cfg, ref64.collider_params(spec), t, nodes)["x"][0]
        idx = np.clip(np.round(x / dx).astype(np.int64), 0, N - 1)
        near |= np.abs(sdf[idx[:, 0], idx[:, 1], idx[:, 2]]) < 2 * dx
    cand = np.unique(nodes[near] >> 2, axis=0)
    keys = [cand[rng.permutation(len(cand))[:48]]] if len(cand) else []
    keys += [np.asarray(centres, np.int64).reshape(-1, 3)]
    ks = rng.integers(0, G, (12, 3))
    ks[:4, 1] = G - 1
    ks[4:8, 0] = 0
    keys = np.unique(np.concatenate(keys + [ks]), axis=0).astype(np.int32)
    nb = len(keys)
    m = np.exp(rng.uniform(np.log(1e-12), 0.0, (nb, 64)))
    u = rng.uniform(size=(nb, 64))
    m[u < 0.1] = 0.0
    m[(u >= 0.1) & (u < 0.15)] = 1e-39                              # subnormal: no mass for the grid update
    v = rng.normal(0.0, 2.0, (nb, 3, 64))
    return keys, np.concatenate([m[:, None], m[:, None] * v], 1).astype(np.float32)


def kernel_matrix(run, ob, entry, boundary, motion, label):
    """Every run of one (entry, boundary, motion) at every t through ``run(cfg, keys, grid, dt, collider spec, objects, t)``;
    returns (worst ratio, near nodes, resolved nodes, branches reached away from their margins)."""
    cfg = kernel_config(ob, boundary)
    worst, near, total, branches = 0.0, 0, 0, set()
    dt = 1e-4
    for ti, t in enumerate(TIMES):
        for ri, (rl, spec, objs) in enumerate(entry_runs(entry, motion)):
            if ri % 3 == 0:   # one grid per shape and t (its surface does not depend on the type)
                keys, grid = synthetic_grid(cfg, objs, spec, t, seed=ti + 10 * boundary + 100 * ENTRIES.index(entry))
            post, mx = run(cfg, keys, grid, dt, spec, objs, t)
            ccol = None
            if spec is not None:
                sdf, grad = S.make_field(cfg.domain_bits, FIELDS["sphere"])
                ccol = (ref64.collider_params(spec), sdf, grad)
            w, n, tot, br = check_collider_update(cfg, keys.astype(np.int64), grid, post, mx, dt, ccol, t, f"{label} {rl} t {t}", objects=objs)
            worst, near, total, branches = max(worst, w), near + n, total + tot, branches | br
    assert near <= MAX_NEAR_NODES * total, f"{label}: {near} of {total} resolved nodes near a discontinuity"
    return worst, near, total, branches


def oracle_kernel(ob):
    import collider_oracle_binding as cob

    def run(cfg, keys, grid, dt, spec, objs, t):
        col = None
        if spec is not None:
            sdf, grad = S.make_field(cfg.domain_bits, FIELDS["sphere"])
            field = block_field(cfg.domain_bits, sdf, grad)
            col = S.collider_struct(cob.Collider(), spec)
            col.sdf = field.ctypes.data
        g = np.ascontiguousarray(grid.copy())
        k = np.ascontiguousarray(keys.reshape(-1))
        part = ob.Partition()
        part.active_keys = k.ctypes.data
        mv = np.zeros(1, np.float32)
        cob.lib().orc_update_grid_velocity_query_max_boundaries(C.byref(cfg), len(keys), ob.ptr(g), part, dt, C.byref(col) if col is not None else None,
                                                                cob.unit_planes(objs), len(objs), np.float32(t), ob.ptr(mv))
        return g, float(mv[0])
    return run


@pytest.mark.parametrize("entry,boundary,motion", KERNEL_MATRIX, ids=[f"{e}-b{b}-{m}" for e, b, m in KERNEL_MATRIX])
def test_oracle_objects_kernel_matches_ref64(oracle, entry, boundary, motion):
    worst, near, total, _ = kernel_matrix(oracle_kernel(oracle), oracle, entry, boundary, motion, f"oracle {entry} boundary {boundary} {motion}")
    print(f"oracle {entry} boundary {boundary} {motion}: worst {worst:.3f} x COLLIDER_VEL_KAPPA, {near} of {total} nodes near")


def test_objects_kernel_reaches_every_branch(oracle):
    """Across the kernel-level matrix, every branch of every shape and of the response is taken by some node away from its
    margins."""
    run = oracle_kernel(oracle)
    got = set()
    for entry, boundary, motion in KERNEL_MATRIX:
        if entry in SHAPES:
            got |= kernel_matrix(run, oracle, entry, boundary, motion, f"{entry} {boundary} {motion}")[3]
    want = {"miss", "plane", "sphere", "sphere_zero", "cyl_cap-", "cyl_cap+", "cyl_side", "cyl_side_tie", "cyl_zero", "sticky", "slip", "slip_friction", "slip_stick",
            "separate_approach", "separate_separate", "zero_normal"} | {f"box_{a}{s}" for a in "xyz" for s in "-+"}
    assert want <= got, f"branches never reached away from a margin: {sorted(want - got)}"


# ---- per sub-step: the oracle with the objects through OBJECT_CASES --------------------------------------------------------
@pytest.mark.parametrize("name", list(S.OBJECT_CASES))
def test_ref64_object_cases_match_oracle(oracle, name):
    oracle_substep_check(oracle, S.OBJECT_CASES[name], name)


def test_object_cases_act():
    """The cases exercise what they are named for: the objects resolve nodes with mass away from their margins, the lattice box
    takes exact ties, the paddle's dt is CFL-bound and set by a node it resolved, the last of the 16 objects touches material,
    list order matters where the objects overlap."""
    import oracle_binding as ob
    want = {"obj_floor_fc_sticky": "sticky", "obj_tilted_plane_slip": "plane", "obj_sphere_separate": "separate_approach", "obj_cylinder_tilted": "cyl_side",
            "obj_lattice_box": "box_y+", "obj_lattice_cylinder": "cyl_side_tie", "obj_paddle_combined": "slip_friction", "obj_top_boundary0": "sticky", "obj_wall_band": "slip_friction"}
    for name, case in S.OBJECT_CASES.items():
        osim = S.build_oracle(ob, case)
        osim.step(case["steps"][-1])
        _, nbc, _ = osim.block_counts()
        nm = len(case["models"])
        objs = S.ref_objects(case)
        r = ref64.substep(osim.cfg, ref_models(case, [osim.particle_state(i) for i in range(nm)]), osim.active_keys()[:nbc], osim.grid(), osim.dt,
                          case["dt"], np.inf, S.ref_collider(case), np.float32(osim.sim_time), objects=objs)
        info = r["collider_info"]
        away = ~info["near"] & (info["branch"] != "")
        got = set(info["branch"][away].tolist()) | set(info["shape_branch"][away].tolist())
        hits = [int((st["hit"] & ~st["near"]).sum()) for st in info["stages"]]
        assert hits[-1] > 0, f"{name}: the last object must touch material away from its margins ({hits})"
        if name in want:
            assert want[name] in got, (name, sorted(got))
        if name == "obj_cylinder_tilted":
            assert {"cyl_cap+", "cyl_side"} <= got, sorted(got)
        if name == "obj_paddle_combined":
            assert r["new_dt"] < case["dt"], "the paddle's dt must be CFL-bound"
            vsq = (r["vel"] ** 2).sum(1)
            b, c = np.unravel_index(np.argmax(vsq), vsq.shape)
            assert info["branch"][b, c] in ("slip", "slip_friction", "slip_stick"), info["branch"][b, c]
        if name == "obj_overlap":
            u = ref64.grid_update(osim.cfg, osim.active_keys()[:nbc], osim.grid(), osim.dt, None, np.float32(osim.sim_time), objs[::-1])
            assert np.abs(u[0] - r["vel"]).max() > 0.1, "the reversed list must give other velocities"
        if name in ("obj_lattice_box", "obj_lattice_cylinder"):
            assert info["near"].sum() == 0, "a static lattice-aligned object decides every tie exactly"
        if name == "obj_top_boundary0":
            keys = osim.active_keys()[:nbc].astype(np.int64)
            top = (keys[:, None, 1] * 4 + ref64._CELLS[None, :, 1] == 63) & (osim.grid()[:, 0] > 0)
            assert (top & (info["branch"] == "sticky")).any(), "a node at 4G - 1 must be resolved"
        osim.close()

