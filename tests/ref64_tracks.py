"""float64 restatement of collision-object motion tracks (DESIGN.md section 2.14) on top of ref64's boundary chain.

    prepare(keys, flags)               the records cb200_track_prepare writes (numpy, double), or ValueError on a rejection
    evaluate(records, flags, t)        pose and kinematic velocity: dict(c, q, v, w, seg, tw) at the float32 time t
    frame(o, t)                        the tracked object's frame in collider_frame's form, each part as (value, E)
    object_resolve(cfg, o, t, ...)     ref64.object_resolve for an object with a track (object_params' "track")
    pivot(o, t)                        (c(t), its E): the pivot of the force report's torque
    boundary_impulses(...)             ref64_forces.boundary_impulses with a tracked body's torque about c(t)
    tracked()                          context in which ref64's chain and ref64_forces move tracked objects on their tracks

As on the device, the periodic wrap, the segment search and u are float32 (t' = t0 + fmodf(t - t0, tn - t0) for t >= tn, the segment
by float compares, u = (t' - t_k) / (t_{k+1} - t_k) in float32); everything after u is float64.  The E of the FP32 frame (units of
2^-24, first order): c(t) 4 (|c_k| + |c_{k+1}|) linear, 16 (|c_k| + |c_{k+1}| + h |m_k| + h |m_{k+1}|) smooth; c'(t) the same / h;
each quaternion component 16 (sinf / cosf within 4 ulp, the sqrt, the product); R = Q R0 64 sum_k |R0_kj|; omega 16 |r| / h.
"""
import contextlib

import numpy as np

import ref64
import ref64_forces as RF

EPS32 = ref64.EPS32
TRACK_SMOOTH, TRACK_PERIODIC = 1, 2


def _keys_array(keys):
    """[(t, pos[3], rot[4])] float32 values from a ctypes cb200_track_key array or tuples"""
    out = []
    for k in keys:
        if hasattr(k, "pos"):
            out.append((np.float32(k.t), np.asarray(list(k.pos), np.float32), np.asarray(list(k.rot), np.float32)))
        else:
            out.append((np.float32(k[0]), np.asarray(k[1], np.float32).reshape(3), np.asarray(k[2], np.float32).reshape(4)))
    return out


def prepare(keys, flags):
    """records[n, 16] float32 (t, pos, rot, tangent, rotvec, 0, 0) as cb200_track_prepare computes them in double; ValueError
    on every rejection it makes."""
    keys = _keys_array(keys)
    n = len(keys)
    periodic = bool(flags & TRACK_PERIODIC)
    if not 1 <= n <= 4096 or flags & ~(TRACK_SMOOTH | TRACK_PERIODIC) or (periodic and n < 2):
        raise ValueError("key count or flags")
    t = np.array([k[0] for k in keys], np.float64)
    c = np.array([k[1] for k in keys], np.float64)
    raw = np.array([k[2] for k in keys], np.float64)
    if not (np.isfinite(t).all() and np.isfinite(c).all() and np.isfinite(raw).all()):
        raise ValueError("non-finite")
    if (np.diff(t) <= 0).any():
        raise ValueError("times not increasing")
    nn = (raw ** 2).sum(1)
    if not (nn > 0).all():
        raise ValueError("zero quaternion")
    q = raw / np.sqrt(nn)[:, None]
    if periodic:
        if not np.array_equal(c[0], c[-1]):
            raise ValueError("periodic position mismatch")
        a, b = q[0].astype(np.float32), q[-1].astype(np.float32)
        if not (np.array_equal(a, b) or np.array_equal(a, (-q[-1]).astype(np.float32))):
            raise ValueError("periodic rotation mismatch")
    for k in range(1, n):
        d = q[k - 1][0] * q[k][0] + q[k - 1][1] * q[k][1] + q[k - 1][2] * q[k][2] + q[k - 1][3] * q[k][3]
        if d == 0.0:
            raise ValueError("antipodal neighbours")
        if d < 0:
            q[k] = -q[k]
    rec = np.zeros((n, 16), np.float64)
    rec[:, 0], rec[:, 1:4], rec[:, 4:8] = t, c, q
    if flags & TRACK_SMOOTH and n > 1:
        for k in range(n):
            if periodic and k in (0, n - 1):
                lo, hi, span = n - 2, 1, (t[1] - t[0]) + (t[n - 1] - t[n - 2])
            else:
                lo, hi = max(k - 1, 0), min(k + 1, n - 1)
                span = t[hi] - t[lo]
            rec[k, 8:11] = (c[hi] - c[lo]) / span
    for k in range(n - 1):
        r = qmul(qconj(q[k]), q[k + 1])
        sn = np.sqrt((r[1:] ** 2).sum())
        if sn > 0:
            rec[k, 11:14] = r[1:] / sn * 2.0 * np.arctan2(sn, r[0])
    return rec.astype(np.float32)


def qconj(q):
    return np.array([q[0], -q[1], -q[2], -q[3]])


def qmul(a, b):
    return np.array([a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                     a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1], a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0]])


def quat_mat(q):
    """row-major rotation matrix of q (not renormalised: the device's formula)"""
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def evaluate(rec, flags, t):
    """The pose at the float32 time t of the float32 records rec[n, 16]: dict(c, q, v (c'), w (world omega), seg (segment or -1 when
    holding), tw (the wrapped float32 time), u, h, key) in float64 after the float32 wrap, search and u."""
    rec = np.asarray(rec, np.float32)
    n = len(rec)
    f = np.float32
    t = f(t)
    t0, tn = rec[0, 0], rec[n - 1, 0]
    if flags & TRACK_PERIODIC and n > 1 and t >= tn:
        t = f(t0 + f(np.fmod(f(t - t0), f(tn - t0))))
    if n > 1 and t0 <= t < tn:
        lo, hi = 0, n - 1
        while hi - lo > 1:
            mid = (lo + hi) // 2
            if t >= rec[mid, 0]:
                lo = mid
            else:
                hi = mid
        h32 = f(rec[lo + 1, 0] - rec[lo, 0])
        u = float(f(f(t - rec[lo, 0]) / h32))
        h = float(h32)
        a, b = rec[lo].astype(np.float64), rec[lo + 1].astype(np.float64)
        ck, c1, mk, m1 = a[1:4], b[1:4], a[8:11], b[8:11]
        if flags & TRACK_SMOOTH:
            h00, h10, h01, h11 = 2 * u ** 3 - 3 * u ** 2 + 1, u ** 3 - 2 * u ** 2 + u, 3 * u ** 2 - 2 * u ** 3, u ** 3 - u ** 2
            d00, d10, d11 = 6 * u ** 2 - 6 * u, 3 * u ** 2 - 4 * u + 1, 3 * u ** 2 - 2 * u
            c = h00 * ck + h10 * h * mk + h01 * c1 + h11 * h * m1
            v = d00 * (ck - c1) / h + d10 * mk + d11 * m1
        else:
            c = ck + u * (c1 - ck)
            v = (c1 - ck) / h
        r = a[11:14]
        th = np.sqrt((r ** 2).sum())
        e = np.array([1.0, 0.0, 0.0, 0.0]) if th == 0 else np.concatenate([[np.cos(0.5 * u * th)], r * np.sin(0.5 * u * th) / th])
        q = qmul(a[4:8], e)
        w = quat_mat(a[4:8]) @ r / h
        return dict(c=c, q=q, v=v, w=w, seg=lo, tw=float(t), u=u, h=h, key=(a, b))
    k = n - 1 if n > 1 and t >= tn else 0
    a = rec[k].astype(np.float64)
    return dict(c=a[1:4].copy(), q=a[4:8].copy(), v=np.zeros(3), w=np.zeros(3), seg=-1, tw=float(t), u=0.0, h=0.0, key=(a, a))


def _prepared(track):
    """(records, flags) of an objects.Track, prepared once"""
    if not hasattr(track, "_ref64_records"):
        track._ref64_records = prepare(track.keys, track.flags)
    return track._ref64_records, track.flags


def _errors(e, flags):
    """E (units of 2^-24) of c, v, q, omega (module docstring)"""
    a, b = e["key"]
    if e["seg"] < 0:
        return np.zeros(3), np.zeros(3), np.zeros(4), np.zeros(3)
    h = e["h"]
    cc = np.abs(a[1:4]) + np.abs(b[1:4])
    if flags & TRACK_SMOOTH:
        ec = 16 * (cc + h * (np.abs(a[8:11]) + np.abs(b[8:11])))
        ev = ec / h
    else:
        ec, ev = 4 * cc, 4 * cc / h
    eq = np.full(4, 16.0)
    ew = np.full(3, 16 * np.sqrt((a[11:14] ** 2).sum()) / h)
    return ec, ev, eq, ew


def frame(o, t):
    """The frame of the tracked object o (object_params with "track") at the float32 time t, in collider_frame's form: rot (9, element
    (i, j) of the material-from-world matrix at 3i + j) = (Q(t) R0)^T as the device stores it, b = c(t), s_inv = 1; plus the track's
    evaluation (track) and the E of its velocities (ev, ew)."""
    rec, flags = _prepared(o["track"])
    e = evaluate(rec, flags, t)
    ec, ev, eq, ew = _errors(e, flags)
    R0 = np.asarray(o["rot_mat"], np.float64).reshape(3, 3).T            # world-from-material: element (k, j) = rot_mat[3j + k]
    W = quat_mat(e["q"]) @ R0
    er = 64.0 * np.broadcast_to(np.abs(R0).sum(0), (3, 3))                # element (i, j): 64 sum_k |R0_kj|
    # rot[3d + j] = M(d, j) with M = W^T: rot[3j + i] = W(i, j)
    rot = W.T.reshape(9)
    erot = er.T.reshape(9)
    return dict(rot=(rot, erot), b=(e["c"], ec), s_inv=ref64._exact(1.0), t=float(np.float32(t)), col=o, track=e, ev=ev, ew=ew)


def material_point(cfg, o, t, nodes):
    """ref64.material_point of the tracked object o at the float32 time t: the same x = R (p - b) s_inv scale + trans on frame(o, t)."""
    f = frame(o, t)
    points = np.asarray(nodes, np.int64).reshape(-1, 3) * (1.0 / (1 << cfg.domain_bits))
    n = len(points)
    R = f["rot"]
    Rb = (np.broadcast_to(R[0], (n, 9)), np.broadcast_to(R[1], (n, 9)))
    xm = ref64._sub(ref64._exact(points), (np.broadcast_to(f["b"][0], (n, 3)), np.broadcast_to(f["b"][1], (n, 3))))
    y = [ref64._dot3(Rb, xm, lambda k, d=d: 3 * d + k, lambda k: k) for d in range(3)]   # s_inv = 1 exactly
    y = (np.stack([c[0] for c in y], -1), np.stack([c[1] for c in y], -1))
    x = ref64._add(ref64._mul(y, ref64._exact(o["scale"])), ref64._exact(o["trans"]))
    return dict(f=f, col=o, Rb=Rb, xm=xm, x=x)


def object_resolve(cfg, o, t, nodes, v, vmag):
    """ref64.object_resolve for an object with a track: its frame (frame), the same query and response, with the rigid object
    velocity vo = c'(t) + omega(t) x (p - c(t)).

    The response is taken from ref64.resolve_query with the object at rest (a tracked object has no omega, trans_vel or dsdt, so its
    reference velocity is exactly 0) on v - vo, and vo added back: the device resolves v - vo and adds vo back in the same way.  The one
    exception is SEPARATE's zero normal, which returns 0 before vo is added back.  Nodes the object does not hit keep v as it is, and the
    |v|^2 range of the near nodes is formed as resolve_query forms it."""
    p = material_point(cfg, o, t, nodes)
    xm, e, f = p["xm"], p["f"]["track"], p["f"]
    n = len(xm[0])
    wv = (np.broadcast_to(e["w"], (n, 3)), np.broadcast_to(f["ew"], (n, 3)))
    cross = [ref64._sub(ref64._mul((wv[0][:, a], wv[1][:, a]), (xm[0][:, b], xm[1][:, b])), ref64._mul((wv[0][:, b], wv[1][:, b]), (xm[0][:, a], xm[1][:, a])))
             for a, b in ((1, 2), (2, 0), (0, 1))]
    cr = (np.stack([c[0] for c in cross], -1), np.stack([c[1] for c in cross], -1))
    vo = ref64._add((np.broadcast_to(e["v"], (n, 3)), np.broadcast_to(f["ev"], (n, 3))), cr)
    vin = (np.asarray(v, np.float64).reshape(n, 3), np.asarray(vmag, np.float64).reshape(n, 3))
    q = ref64.object_query(o, p["x"])
    rel = ref64._sub(vin, vo)
    r = ref64.resolve_query(p, q, rel[0], rel[1])
    hit = r["hit"]
    gone = (q["zero"] & hit)[:, None] if o["type"] == ref64.SEPARATE else np.zeros((n, 1), bool)
    back = ref64._add((r["res_v"], r["mag"]), vo)
    res_v = np.where(gone, 0.0, back[0])
    res_e = np.where(gone, 0.0, back[1])
    out_v = np.where(hit[:, None], res_v, vin[0])
    out_e = np.where(hit[:, None], res_e, vin[1])
    near, span = r["near"], r["span"]
    ovo = np.sqrt((vo[0] ** 2).sum(1))
    vsq, alt_hit, alt_miss = (out_v ** 2).sum(1), (res_v ** 2).sum(1), (vin[0] ** 2).sum(1)
    lo = np.where(near, np.minimum(alt_hit, alt_miss), vsq)
    hi = np.where(near, np.maximum(alt_hit, alt_miss), vsq)
    if o["type"] != ref64.STICKY:
        za = r["normal_alt"]
        lo = np.where(za, np.minimum(lo, np.maximum(ovo - span, 0.0) ** 2), lo)
        hi = np.where(za, np.maximum(hi, (ovo + span) ** 2), hi)
    return dict(r, v=out_v, mag=out_e, vo=vo[0], vsq_lo=lo, vsq_hi=hi, res_v=res_v, ovo=ovo)


def pivot(o, t):
    """(c(t), E of its FP32 value) of the tracked object o (object_params with "track") at the float32 time t"""
    rec, flags = _prepared(o["track"])
    e = evaluate(rec, flags, t)
    return e["c"], _errors(e, flags)[0]


# ---- tracked objects inside ref64's chain ---------------------------------------------------------------------------------------
_OBJECT_PARAMS, _OBJECT_RESOLVE, _BOUNDARY_IMPULSES = ref64.object_params, ref64.object_resolve, RF.boundary_impulses


def object_params(o):
    """ref64.object_params, keeping the object's track (the "track" of claymore_b200.objects' track= keyword, or a dict's)"""
    p = _OBJECT_PARAMS(o)
    track = o.get("track") if isinstance(o, dict) else getattr(o, "track", None)
    if track is not None:
        p["track"] = track
    return p


def _object_resolve(cfg, o, t, nodes, v, vmag):
    if o.get("track") is None:
        return _OBJECT_RESOLVE(cfg, o, t, nodes, v, vmag)
    return object_resolve(cfg, o, t, nodes, v, vmag)


def boundary_impulses(cfg, keys, grid, dt, collider=None, t=0.0, objects=None):
    """ref64_forces.boundary_impulses with a tracked body's pivot c(t) (pivot) and that pivot's E in the bound of L; untracked bodies as
    there (b(t) = trans + trans_vel t)."""
    keys = np.asarray(keys, np.int64)
    objects = [ref64.object_params(o) for o in objects] if objects else []
    has, m, v, mag = RF.pre_chain_velocity(cfg, keys, grid, dt)
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
    t32 = float(np.float32(t))
    for k, prm, st in stages:
        r = st(nodes, cur, cmag)
        out, omag = r["v"], r["mag"]
        dj = mass[:, None] * (cur - out)
        if prm.get("track") is not None:
            piv, piv_e = pivot(prm, t)
            piv_e = piv_e.sum()
        else:
            piv = np.asarray(prm["trans"], np.float64) + np.asarray(prm["trans_vel"], np.float64) * t32
            piv_e = np.abs(prm["trans"]).sum() + 2 * np.abs(np.asarray(prm["trans_vel"]) * t32).sum()
        xm = p - piv
        J[k] = dj.sum(0)
        L[k] = np.cross(xm, dj).sum(0)
        rxm = np.sqrt((xm ** 2).sum(1))
        tainted |= r["near"]
        fr = abs(prm["friction"])
        vo = np.sqrt((r["vo"] ** 2).sum(1))
        S_out = np.maximum(S, (2 + fr) * vo + (1 + fr) * S) * (1 + 8 * EPS32)
        e = mass * ((cmag + omag).sum(1)) * RF.VEL_KAPPA * EPS32
        e = np.where(tainted, 0.0, e)
        w = np.where(tainted, 2 * mass * (S + S_out), 0.0)
        adj = np.abs(dj)
        xm_err = EPS32 * (2 * rxm + piv_e)
        bJ[k] = (e + w).sum() + RF.SUM_ULPS * EPS32 * adj.sum(0)
        bL[k] = (2 * e * rxm + w * (rxm + 2 * dx) + 2 * adj.sum(1) * xm_err).sum() + RF.CROSS_ULPS * EPS32 * (rxm[:, None] * adj).sum(0)
        cur, cmag, S = out, omag, S_out
    return dict(J=J, L=L, bJ=bJ, bL=bL, near=tainted, nodes=len(nodes))


@contextlib.contextmanager
def tracked():
    """ref64 and ref64_forces with tracked objects: object_params keeps an object's track, object_resolve moves a tracked object on it
    (object_resolve above), ref64_forces.boundary_impulses takes a tracked body's torque about c(t); everything that calls them
    (object_chain, grid_update, substep, the MGSP reference, the sub-step loops) follows.  Restored on exit."""
    ref64.object_params, ref64.object_resolve, RF.boundary_impulses = object_params, _object_resolve, boundary_impulses
    try:
        yield
    finally:
        ref64.object_params, ref64.object_resolve, RF.boundary_impulses = _OBJECT_PARAMS, _OBJECT_RESOLVE, _BOUNDARY_IMPULSES
