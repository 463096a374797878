"""The signed-distance collider against the float64 reference (ref64.collider_resolve), per node, per sub-step and in the dt.

Kernel level: orc_update_grid_velocity_query_max_collider on synthetic grids (blocks around each field's surface, masses
log-uniform from 1e-12 to 1 with zero and subnormal nodes, velocities N(0, 2) m/s) over 3 types x friction {0, 0.3, -0.2} x
{static, combined motion} x t {0, 0.37, 3.1} x {sphere, box, tilted plane, zero-gradient slab} x boundary {2, 0}; friction
-0.2 separates SLIP's `friction > 0` from SEPARATE's `friction != 0`.  Per node: |v - ref64| <= COLLIDER_VEL_KAPPA 2^-24 E,
nodes near a discontinuity (ref64's margin) left out and counted.  Per sub-step: the collider oracle through COLLIDER_CASES
with ref64_checks' single-domain kappa (F excepted, COLLIDER_KAPPA); particles that read a near node and the cells
they write are left out and counted, each under its cap.  The GPU tests (test_gpu_collider_ref64.py) hold the engine to the same values.
"""
import ctypes as C

import numpy as np
import pytest

import ref64
import ref64_cases as S
from ref64_checks import COLLIDER_VEL_KAPPA, MAX_NEAR_NODES, oracle_substep_check, ref_models

COLLIDER_MAX_REL = 4.0     # the max |v|^2 within 4 x 2^-24 relative of [mx_lo, mx_hi] (the near nodes' branch choices)

DOMAIN_BITS = 6
FIELDS = {
    "sphere": ("sphere", (0.52, 0.47, 0.5), 0.21),
    "box": ("box", (0.3, 0.28, 0.33), (0.68, 0.61, 0.7)),
    "tilted_plane": ("plane", (0.5, 0.55, 0.5), (0.3, -1.0, 0.2)),     # solid above: reaches the top face
    "zero_slab": ("zero_slab", 0.4),
}


def _rot(ax, ay, az):
    cx, sx, cy, sy, cz, sz = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay), np.cos(az), np.sin(az)
    return np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]]) @ np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])


MOTIONS = {
    "static": dict(),
    # every motion at once, about a point near the fields' centres so that the object stays in the domain up to t = 3.1
    "combined": dict(rot_mat=_rot(0.3, -0.2, 0.5), trans=(0.5, 0.47, 0.5), trans_vel=(0.04, -0.03, 0.02), omega=(0.3, -0.2, 0.5), scale=1.15, dsdt=0.2),
}
TYPES = (S.STICKY, S.SLIP, S.SEPARATE)
FRICTIONS = (0.0, 0.3, -0.2)
TIMES = (0.0, 0.37, 3.1)
KERNEL_MATRIX = [(f, b, m) for f in FIELDS for b in (2, 0) for m in MOTIONS]


def kernel_config(ob, boundary):
    return ob.make_config(domain_bits=DOMAIN_BITS, boundary=boundary)


def collider_of(typ, friction, motion, field="sphere"):
    return dict(field=FIELDS[field], type=typ, friction=friction, **MOTIONS[motion])


def block_field(domain_bits, sdf, grad):
    """the level set in the engine's layout: G^3 blocks row-major, each [4][64] (distance, gradient x, y, z)"""
    g = 1 << (domain_bits - 2)
    a = np.concatenate([sdf[None], grad]).reshape(4, g, 4, g, 4, g, 4)
    return np.ascontiguousarray(a.transpose(1, 3, 5, 0, 2, 4, 6).reshape(-1)).astype(np.float32)


def synthetic_grid(cfg, field, motion, t, seed):
    """(keys[nb, 3] int32, grid[nb, 4, 64] float32): up to 48 blocks whose nodes lie within 2 dx of the surface of ``field``
    (placed by ``motion`` at t), 4 blocks at the top face, 4 at the low x face and 4 anywhere."""
    rng = np.random.default_rng(seed)
    G = 1 << (cfg.domain_bits - 2)
    N, dx = 4 * G, 1.0 / (1 << cfg.domain_bits)
    sdf, _ = S.make_field(cfg.domain_bits, FIELDS[field])
    f = ref64.collider_frame(ref64.collider_params(S.collider_spec(collider_of(0, 0.0, motion, field))), t)
    A = f["rot"][0].reshape(3, 3)
    nodes = np.stack(np.meshgrid(*[np.arange(N)] * 3, indexing="ij"), -1).reshape(-1, 3)
    col = ref64.collider_params(S.collider_spec(collider_of(0, 0.0, motion, field)))
    x = ((nodes * dx - f["b"][0]) * f["s_inv"][0]) @ A.T * col["scale"] + col["trans"]
    idx = np.clip(np.round(x / dx).astype(np.int64), 0, N - 1)
    near = np.abs(sdf[idx[:, 0], idx[:, 1], idx[:, 2]]) < 2 * dx
    cand = np.unique(nodes[near] >> 2, axis=0)
    keys = [cand[rng.permutation(len(cand))[:48]]] if len(cand) else []
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
    grid = np.concatenate([m[:, None], m[:, None] * v], 1).astype(np.float32)
    return keys, grid


def oracle_update(cob, ob, cfg, keys, grid, dt, col, t):
    """orc_update_grid_velocity_query_max_collider on copies -> (grid[nb, 4, 64], max |v|^2)"""
    g = np.ascontiguousarray(grid.copy())
    k = np.ascontiguousarray(keys.reshape(-1))
    part = ob.Partition()
    part.active_keys = k.ctypes.data
    mv = np.zeros(1, np.float32)
    cob.lib().orc_update_grid_velocity_query_max_collider(C.byref(cfg), len(keys), ob.ptr(g), part, dt, C.byref(col), np.float32(t), ob.ptr(mv))
    return g, float(mv[0])


def check_collider_update(cfg, keys, pre, post, mx_impl, dt, ccol, t, label, objects=None):
    """One implementation's collider grid update (``ccol`` = (col, sdf, grad) or None, then ``objects``) against ref64 ->
    (worst ratio, near nodes, resolved nodes, branches away; with objects also each shape's branches, per list entry)."""
    vel, vmag, mx, info = ref64.grid_update(cfg, keys, pre.astype(np.float64), dt, ccol, t, objects)
    post = np.asarray(post, np.float64)
    assert np.array_equal(post[:, 0], pre[:, 0]), f"{label}: the grid update changed the mass channel"
    has = pre[:, 0] >= ref64.FLT_MIN32
    near = info["near"]
    err = np.abs(post[:, 1:] - vel)
    bound = COLLIDER_VEL_KAPPA * ref64.EPS32 * vmag
    ok = (err <= bound) | near[:, None, :]
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(err > 0, err / bound, 0.0)
    ratio = np.where(near[:, None, :], 0.0, np.nan_to_num(ratio, nan=np.inf))
    if not ok.all():
        b, d, c = np.unravel_index(np.argmax(ratio), ratio.shape)
        node = tuple(int(v) for v in keys[b] * 4 + ref64._CELLS[c])
        raise AssertionError(f"{label}: node {node} ({info['branch'][b, c]}) component {d}: {post[b, 1 + d, c]!r} vs ref64 {vel[b, d, c]!r}, "
                             f"{ratio[b, d, c]:.3g} x its bound (E {vmag[b, d, c]:.3g}, object velocity {info['vo'][b, :, c]})")
    # the max: 4 x 2^-24 relative, widened by what the velocities' own bounds allow a node's |v|^2 (at a box's edge E can
    # exceed |v|: the normal moves with the last bit of the material-space point)
    dv = COLLIDER_VEL_KAPPA * ref64.EPS32 * vmag
    slack = float(np.where(has & ~near, (2 * np.abs(vel) * dv + dv ** 2).sum(1), 0.0).max(initial=0.0))
    lo = info["mx_lo"] * (1 - COLLIDER_MAX_REL * ref64.EPS32) - slack
    hi = info["mx_hi"] * (1 + COLLIDER_MAX_REL * ref64.EPS32) + slack
    assert lo <= mx_impl <= hi, f"{label}: max |v|^2 {mx_impl!r} outside [{info['mx_lo']!r}, {info['mx_hi']!r}] (ref64 {mx!r}, slack {slack:.3g})"
    away = has & ~near
    branches = set(info["branch"][away].tolist())
    for st in info.get("stages", ()):
        on = has & st["hit"] & ~st["near"]
        branches |= set(st["branch"][on].tolist()) | set(st["shape_branch"][on].tolist())
    return float(ratio.max(initial=0.0)), int((near & has).sum()), int(has.sum()), branches


def kernel_matrix(run, ob, field, boundary, motion, label):
    """Every type, friction and time of one (field, boundary, motion) through ``run(cfg, keys, grid, dt, col_params, t)``;
    returns (worst ratio, near nodes, resolved nodes, branches reached away from their margins)."""
    cfg = kernel_config(ob, boundary)
    worst, near, total, branches = 0.0, 0, 0, set()
    dt = 1e-4
    for ti, t in enumerate(TIMES):
        keys, grid = synthetic_grid(cfg, field, motion, t, seed=ti + 10 * boundary + 100 * list(FIELDS).index(field))
        sdf, grad = S.make_field(cfg.domain_bits, FIELDS[field])
        for typ in TYPES:
            for fr in FRICTIONS:
                spec = S.collider_spec(collider_of(typ, fr, motion, field))
                post, mx = run(cfg, keys, grid, dt, spec, t)
                ccol = (ref64.collider_params(spec), sdf, grad)
                w, n, tot, br = check_collider_update(cfg, keys.astype(np.int64), grid, post, mx, dt, ccol, t, f"{label} type {typ} friction {fr} t {t}")
                worst, near, total, branches = max(worst, w), near + n, total + tot, branches | br
    assert near <= MAX_NEAR_NODES * total, f"{label}: {near} of {total} resolved nodes near a discontinuity"
    return worst, near, total, branches


def oracle_kernel(ob):
    import collider_oracle_binding as cob

    def run(cfg, keys, grid, dt, spec, t):
        sdf, grad = S.make_field(cfg.domain_bits, spec_field[0])
        field = block_field(cfg.domain_bits, sdf, grad)
        col = S.collider_struct(cob.Collider(), spec)
        col.sdf = field.ctypes.data
        return oracle_update(cob, ob, cfg, keys, grid, dt, col, t)
    spec_field = [None]
    return run, spec_field


@pytest.mark.parametrize("field,boundary,motion", KERNEL_MATRIX, ids=[f"{f}-b{b}-{m}" for f, b, m in KERNEL_MATRIX])
def test_oracle_collider_kernel_matches_ref64(oracle, field, boundary, motion):
    run, spec_field = oracle_kernel(oracle)
    spec_field[0] = FIELDS[field]
    worst, near, total, _ = kernel_matrix(run, oracle, field, boundary, motion, f"oracle {field} boundary {boundary} {motion}")
    print(f"oracle {field} boundary {boundary} {motion}: worst {worst:.3f} x COLLIDER_VEL_KAPPA, {near} of {total} nodes near")


def test_collider_kernel_reaches_every_branch(oracle):
    """Across the kernel-level matrix, every branch of the collider is taken by some node away from its margins."""
    run, spec_field = oracle_kernel(oracle)
    got = set()
    for field, boundary, motion in KERNEL_MATRIX:
        spec_field[0] = FIELDS[field]
        got |= kernel_matrix(run, oracle, field, boundary, motion, f"{field} {boundary} {motion}")[3]
    want = {"miss", "band", "top", "sticky", "slip", "slip_friction", "slip_stick", "separate_approach", "separate_separate", "zero_normal"}
    assert want <= got, f"branches never reached away from a margin: {sorted(want - got)}"


# ---- per sub-step: the collider oracle through COLLIDER_CASES ---------------------------------------------------------------
@pytest.mark.parametrize("name", list(S.COLLIDER_CASES))
def test_ref64_collider_cases_match_oracle(oracle, name):
    oracle_substep_check(oracle, S.COLLIDER_CASES[name], name)


def test_collider_cases_act():
    """The cases exercise what they are named for: the floor and paddle cases resolve nodes, the paddle's dt is CFL-bound and
    set by a node the collider resolved, the thin-wall case has mass on nodes whose cell's +1 node is 4G, the zero-gradient
    cases take the zero-normal branch."""
    import oracle_binding as ob
    for name, want in (("floor_fc_sticky", "sticky"), ("paddle_combined", "slip_friction"), ("zero_grad_slip", "zero_normal"),
                       ("zero_grad_separate", "zero_normal"), ("thin_top_boundary0", "top"), ("walls_solid", "band"), ("sphere_separate", "separate_approach")):
        case = S.COLLIDER_CASES[name]
        osim = S.build_oracle(ob, case)
        osim.step(case["steps"][-1])
        _, nbc, _ = osim.block_counts()
        nm = len(case["models"])
        r = ref64.substep(osim.cfg, ref_models(case, [osim.particle_state(i) for i in range(nm)]), osim.active_keys()[:nbc], osim.grid(), osim.dt,
                          case["dt"], np.inf, S.ref_collider(case), np.float32(osim.sim_time))
        info = r["collider_info"]
        assert want in set(info["branch"][~info["near"]].tolist()), (name, set(info["branch"].ravel().tolist()))
        if name == "paddle_combined":
            assert r["new_dt"] < case["dt"], "the paddle's dt must be CFL-bound"
            vel = r["vel"]
            vsq = (vel ** 2).sum(1)
            b, c = np.unravel_index(np.argmax(vsq), vsq.shape)
            assert info["branch"][b, c] in ("slip", "slip_friction", "slip_stick"), info["branch"][b, c]
        osim.close()


# ---- identities of the reference's collider ---------------------------------------------------------------------------------
def _random_nodes(rng, n=4000, N=64):
    return rng.integers(8, N - 8, (n, 3)), rng.normal(0, 2, (n, 3))


@pytest.mark.parametrize("motion", list(MOTIONS))
def test_ref64_collider_identities(motion):
    from claymore_b200._capi import Config
    cfg = Config(domain_bits=DOMAIN_BITS, boundary=2)
    rng = np.random.default_rng(3)
    nodes, v = _random_nodes(rng)
    sdf, grad = S.make_field(DOMAIN_BITS, FIELDS["sphere"])
    for t in TIMES:
        out = {}
        for typ in TYPES:
            col = ref64.collider_params(S.collider_spec(collider_of(typ, 0.0, motion)))
            out[typ] = ref64.collider_resolve(cfg, col, sdf, grad, t, nodes, v, np.abs(v))
        hit = out[S.STICKY]["hit"]
        assert hit.sum() > 50 and (~hit).sum() > 50
        # STICKY: v = vo exactly
        assert np.array_equal(out[S.STICKY]["v"][hit], out[S.STICKY]["vo"][hit])
        assert np.array_equal(out[S.STICKY]["v"][~hit], v[~hit])
        # frictionless SLIP: n . (v - vo) = 0, with n the rotated normal; SEPARATE separating: v unchanged
        for typ in (S.SLIP, S.SEPARATE):
            o = out[typ]
            rel = o["v"] - o["vo"]
            if typ == S.SLIP:
                # the projection takes n vn out of v - vo, so what is left is orthogonal to what was taken out: n . (v - vo) = 0
                # up to |n|^2 - 1, which a float32 rot_mat leaves at 1e-7
                removed = (v - o["vo"]) - rel
                dot = np.abs((removed * rel).sum(1))
                assert np.all(dot[hit] <= 1e-6 * (1e-12 + (removed ** 2).sum(1) + (rel ** 2).sum(1))[hit]), motion
            else:
                sep = hit & (o["branch"] == "separate_separate")
                assert sep.sum() > 10
                assert np.allclose(o["v"][sep], v[sep], rtol=0, atol=1e-14)
    # the frame at t = 0 is rot_mat
    col = ref64.collider_params(S.collider_spec(collider_of(S.SLIP, 0.0, motion)))
    f = ref64.collider_frame(col, 0.0)
    assert np.array_equal(f["rot"][0], col["rot_mat"]) and np.all(f["rot"][1] == 0)
