"""float64 restatement of the boundary impulse report (DESIGN.md section 2.13) on top of ref64's boundary chain.

    boundary_impulses(cfg, keys, grid, dt, collider, t, objects)   per-body (J, L) of one grid update and their error bounds
    pre_chain_velocity(cfg, keys, grid, dt)                        the FP32 velocities the chain receives (wall mask, gravity)

Body 0 is the level-set collider (zeros without one), body 1 + i object i.  Each stage is ref64's own collider_resolve /
object_resolve (level-set objects inside ref64_levelset.registered), so v_in / v_out of a body are the velocities the previous
stage left and this one leaves.  J = sum m (v_in - v_out), L = sum (p - b(t)) x m (v_in - v_out), b(t) = trans + trans_vel t.

Bounds, per body and component (2^-24 = EPS32):
  * a node no stage so far has flagged near: m (E_in + E_out) VEL_KAPPA EPS32 in J, times 2 |p - b| in L (E: ref64's error
    magnitudes of the stage's input and output), plus |m dv| times the rounding of p - b in L;
  * a node flagged near at this stage or an earlier one may take any candidate branch from there on: its contribution may be
    anything within m (|dv_ref| + |dv_fp32|) <= 2 m (S_in + S_out), S the largest speed any branch reaches (a stage maps a speed S
    to at most (2 + |friction|) |vo| + (1 + |friction|) S), times |p - b| + 2 dx in L;
  * the FP32 products and the warp sums (two cells, then 5 shuffle levels): SUM_ULPS EPS32 sum |m dv| in J, and CROSS_ULPS EPS32
    sum |p - b| |m dv| in L.
"""
import numpy as np

import ref64

EPS32 = ref64.EPS32
VEL_KAPPA = 4.0    # ref64_checks.COLLIDER_VEL_KAPPA: the per-node velocity bound the resolved grid is held to
SUM_ULPS = 8.0     # product m dv (1) + two-cell add (1) + log2(32) shuffle levels (5) + conversion (1)
CROSS_ULPS = 12.0  # the above + the cross product's two products and difference + the offset


def pre_chain_velocity(cfg, keys, grid, dt):
    """(has[nb, 64], m[nb, 64], v[nb, 3, 64] float64, mag) of ref64.grid_update without boundaries: the velocity the chain receives"""
    v, mag, _ = ref64.grid_update(cfg, keys, grid, dt)
    m = np.asarray(grid, np.float64)[:, 0]
    return m >= ref64.FLT_MIN32, m, v, mag


def _pivot(p, t):
    t = float(np.float32(t))
    return np.asarray(p["trans"], np.float64) + np.asarray(p["trans_vel"], np.float64) * t


def boundary_impulses(cfg, keys, grid, dt, collider=None, t=0.0, objects=None):
    """dict(J[B, 3], L[B, 3], bJ[B, 3], bL[B, 3], near (nodes flagged near anywhere), nodes) for B = 1 + len(objects) bodies, the
    collider = (col, sdf, grad) (ref64 form) or None, the objects cb200_collision_object / object_params, all placed at t."""
    keys = np.asarray(keys, np.int64)
    objects = [ref64.object_params(o) for o in objects] if objects else []
    has, m, v, mag = pre_chain_velocity(cfg, keys, grid, dt)
    b, c = np.nonzero(has)
    nodes = keys[b] * 4 + ref64._CELLS[c]
    mass = m[b, c]
    cur, cmag = v[b, :, c], mag[b, :, c]
    dx = 1.0 / (1 << cfg.domain_bits)
    p = nodes * dx
    stages = []
    if collider is not None:
        col, sdf, grad = collider
        stages.append((0, col, lambda nd, vv, vm: ref64.collider_resolve(cfg, col, sdf, grad, t, nd, vv, vm)))
    for i, o in enumerate(objects):
        stages.append((1 + i, o, lambda nd, vv, vm, o=o: ref64.object_resolve(cfg, o, t, nd, vv, vm)))
    B = 1 + len(objects)
    J, L, bJ, bL = (np.zeros((B, 3)) for _ in range(4))
    tainted = np.zeros(len(nodes), bool)
    S = np.sqrt((cur ** 2).sum(1)) * (1 + 8 * EPS32)
    for k, prm, st in stages:
        r = st(nodes, cur, cmag)
        out, omag = r["v"], r["mag"]
        dj = mass[:, None] * (cur - out)
        xm = p - _pivot(prm, t)
        J[k] = dj.sum(0)
        L[k] = np.cross(xm, dj).sum(0)
        rxm = np.sqrt((xm ** 2).sum(1))
        tainted |= r["near"]
        fr = abs(prm["friction"])
        vo = np.sqrt((r["vo"] ** 2).sum(1))
        S_out = np.maximum(S, (2 + fr) * vo + (1 + fr) * S) * (1 + 8 * EPS32)
        # clean nodes: the FP32 velocities' own error
        e = mass * ((cmag + omag).sum(1)) * VEL_KAPPA * EPS32
        e = np.where(tainted, 0.0, e)
        # any branch from here on
        w = np.where(tainted, 2 * mass * (S + S_out), 0.0)
        adj = np.abs(dj)
        xm_err = EPS32 * (2 * rxm + np.abs(prm["trans"]).sum() + 2 * np.abs(np.asarray(prm["trans_vel"]) * float(np.float32(t))).sum())
        bJ[k] = (e + w).sum() + SUM_ULPS * EPS32 * adj.sum(0)
        bL[k] = (2 * e * rxm + w * (rxm + 2 * dx) + 2 * adj.sum(1) * xm_err).sum() + CROSS_ULPS * EPS32 * (rxm[:, None] * adj).sum(0)
        cur, cmag, S = out, omag, S_out
    return dict(J=J, L=L, bJ=bJ, bL=bL, near=tainted, nodes=len(nodes))
