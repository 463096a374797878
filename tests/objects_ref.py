"""float64 restatement of the analytic collision objects (DESIGN.md section 2.9) for the tests: the grid update's wall mask and
gravity, then each object in list order, placed at time t (the collider's frame and motion model, collider.cuh).

Beside each node's velocity it reports whether the node lies near one of the objects' discontinuities (the hit test, the box's
face tie and its centre sign, the cylinder's cap / side choice, a zero normal), where float32 may take the other branch."""
import numpy as np

STICKY, SLIP, SEPARATE = 0, 1, 2
PLANE, BOX, SPHERE, CYLINDER = 0, 1, 2, 3


def _axis_rot(a, d):
    c, s = np.cos(a), np.sin(a)
    r = np.zeros(9)
    if d == 0:
        r[0], r[4], r[8], r[7], r[5] = 1, c, c, s, -s
    elif d == 1:
        r[4], r[0], r[8], r[2], r[6] = 1, c, c, s, -s
    else:
        r[8], r[0], r[4], r[3], r[1] = 1, c, c, s, -s
    return r


def _mat_mul(a, b):
    c = np.zeros(9)
    for j in range(3):
        for i in range(3):
            c[3 * j + i] = a[i] * b[3 * j] + a[3 + i] * b[3 * j + 1] + a[6 + i] * b[3 * j + 2]
    return c


def params(o):
    """an object's float32 fields as float64 (a cb200_collision_object or a dict with its fields)"""
    get = (lambda k: o[k]) if isinstance(o, dict) else (lambda k: getattr(o, k))
    f = lambda x: np.asarray(np.asarray(x, np.float32), np.float64)   # noqa: E731
    return dict(shape=int(get("shape")), type=int(get("type")), friction=float(f(get("friction"))), a=f(list(get("a"))), b=f(list(get("b"))),
                rot_mat=f(list(get("rot_mat"))), trans=f(list(get("trans"))), trans_vel=f(list(get("trans_vel"))), omega=f(list(get("omega"))),
                dsdt=float(f(get("dsdt"))), scale=float(f(get("scale"))))


def query(o, x, tol):
    """hit[n], normal[n, 3] (material space) and near[n] of object o at the material-space points x[n, 3]"""
    a, b = o["a"], o["b"]
    n = np.zeros_like(x)
    if o["shape"] == PLANE:
        phi = (x - a) @ b
        return phi <= 0, np.broadcast_to(b, x.shape).copy(), np.abs(phi) <= tol
    if o["shape"] == BOX:
        ql, qh = a - x, x - b
        q = np.maximum(ql, qh)
        phi = q.max(1)
        axis = np.argmax(q, 1)
        srt = np.sort(q, 1)
        tie = (srt[:, 2] - srt[:, 1]) <= tol
        sgn = np.where(ql[np.arange(len(x)), axis] > qh[np.arange(len(x)), axis], -1.0, 1.0)
        centre = np.abs(ql[np.arange(len(x)), axis] - qh[np.arange(len(x)), axis]) <= tol
        n[np.arange(len(x)), axis] = sgn
        return phi <= 0, n, (np.abs(phi) <= tol) | ((phi <= 0) & (tie | centre))
    d = x - a
    r = b[0]
    if o["shape"] == SPHERE:
        ln = np.sqrt((d ** 2).sum(1))
        n = np.where(ln[:, None] > 0, d / np.where(ln > 0, ln, 1.0)[:, None], 0.0)
        return ln <= r, n, (np.abs(ln - r) <= tol) | (ln <= tol)
    h = b[1]
    rho = np.sqrt(d[:, 0] ** 2 + d[:, 2] ** 2)
    hit = (rho <= r) & (np.abs(d[:, 1]) <= h)
    phi = np.maximum(rho - r, np.abs(d[:, 1]) - h)
    cap = (h - np.abs(d[:, 1])) < (r - rho)
    n[:, 1] = np.where(cap, np.where(d[:, 1] < 0, -1.0, 1.0), 0.0)
    safe = np.where(rho > 0, rho, 1.0)
    n[:, 0] = np.where(~cap & (rho > 0), d[:, 0] / safe, 0.0)
    n[:, 2] = np.where(~cap & (rho > 0), d[:, 2] / safe, 0.0)
    near = (np.abs(phi) <= tol) | (hit & ((np.abs((h - np.abs(d[:, 1])) - (r - rho)) <= tol) | (rho <= tol) | (cap & (np.abs(d[:, 1]) <= tol))))
    return hit, n, near


def resolve(o, nodes, dx, t, v, tol=1e-5):
    """collider_resolve of the velocities v[n, 3] at grid nodes nodes[n, 3] against object o (params) at time t: (v, near)"""
    cur = o["rot_mat"].copy()
    for d in range(3):
        cur = _mat_mul(cur, _axis_rot(o["omega"][d] * t, d))
    R = cur
    b = o["trans"] + o["trans_vel"] * t
    xm = nodes * dx - b
    x0 = xm / (1.0 + o["dsdt"] * t)
    Rm = R.reshape(3, 3)              # storage (i, j) at 3i + j
    x = (x0 @ Rm.T) * o["scale"] + o["trans"]
    hit, on, near = query(o, x, tol)
    w = o["omega"]
    vo = np.stack([w[1] * xm[:, 2] - w[2] * xm[:, 1], w[2] * xm[:, 0] - w[0] * xm[:, 2], w[0] * xm[:, 1] - w[1] * xm[:, 0]], 1)
    vo += xm * (o["dsdt"] / o["scale"])
    r = x - o["trans"]
    mv = np.stack([w[1] * r[:, 2] + w[2] * r[:, 1], w[2] * r[:, 0] + w[0] * r[:, 2], w[0] * r[:, 1] + w[1] * r[:, 0]], 1) + o["trans_vel"]
    vo += (mv @ Rm) * o["scale"] + o["trans_vel"]
    vr = v - vo
    nrm = on @ Rm
    zero = ~on.any(1)
    typ, fr = o["type"], o["friction"]
    out = v.copy()
    if typ == STICKY:
        res = vo
    else:
        vn = (nrm * vr).sum(1)
        proj = vr - nrm * vn[:, None]
        use = (typ == SLIP) | (vn < 0)
        fric = ((fr > 0) if typ == SLIP else (fr != 0)) & (vn < 0)
        ln = np.sqrt((proj ** 2).sum(1))
        stick = -vn * fr >= ln
        slide = proj + proj / np.where(ln > 0, ln, 1.0)[:, None] * (vn * fr)[:, None]
        f = np.where(fric[:, None], np.where(stick[:, None], 0.0, slide), proj)
        res = np.where(use[:, None], f, vr) + vo
        if typ == SEPARATE:
            res = np.where(zero[:, None], 0.0, res)
    out = np.where(hit[:, None], res, out)
    return out, near


def grid_update(cfg, keys, grid, dt, objs, t):
    """the objects form of the grid update on blocks keys[nb, 3], grid[nb, 4, 64] (float32): (vel[nb, 3, 64], near[nb, 64], max |v|^2
    over the nodes that are not near)"""
    G, bc = 1 << (cfg.domain_bits - 2), cfg.boundary
    dx = 1.0 / (1 << cfg.domain_bits)
    keys = np.asarray(keys, np.int64)
    g = np.asarray(grid, np.float64)
    cells = np.stack(np.meshgrid(np.arange(4), np.arange(4), np.arange(4), indexing="ij"), -1).reshape(64, 3)
    wall = (keys < bc) | (keys >= G - bc)
    m = g[:, 0]
    has = m >= np.finfo(np.float32).tiny
    v = np.where(wall[:, :, None], 0.0, g[:, 1:] / np.where(has, m, 1.0)[:, None])
    v[:, 1] += float(np.float32(cfg.gravity)) * dt
    bi, ci = np.nonzero(has)
    nodes = keys[bi] * 4 + cells[ci]
    vv = v[bi, :, ci]
    near = np.zeros(len(bi), bool)
    for o in objs:
        vv, nr = resolve(params(o), nodes, dx, t, vv)
        near |= nr
    out = np.where(has[:, None], v, g[:, 1:])
    out[bi, :, ci] = vv
    nmap = np.zeros(has.shape, bool)
    nmap[bi, ci] = near
    vsq = (vv ** 2).sum(1)
    return out, nmap, float(vsq[~near].max(initial=0.0)), float(vsq.max(initial=0.0))
