"""float64 restatement of the level-set collision objects (CB200_SHAPE_LEVELSET, DESIGN.md section 2.11) on top of ref64.

    lattice(n, phi)                    the float32 lattice cb200_levelset_prepare builds: float32[nk, nj, ni, 4] (phi, g_i, g_j, g_k)
    levelset_query(o, lat, x)          the query dict ref64.resolve_query takes, with the rounding margins of the box, the hit test
                                       and the zero normal
    registered(lattices)               context in which ref64's object_query, object_chain and grid_update answer CB200_SHAPE_LEVELSET
                                       objects from lattices[b[1]]; every other shape is ref64's own, unchanged
    hits(o, lat, points)               the hit set and its flagged (near) points for world-space float32 points (sinks)

Error terms (ref64's rules): q_d = (x_d - a_d) / c carries E_q = (E_x + rnd(x - a)) / c + rnd(q); t = q - i0 is exact in float32,
1 - t rounds; the trilinear value of each channel has ref64._trilinear's E plus its sensitivity to q, the largest one-sided slope
of the cell and its neighbours (ref64._slope in index units) times E_q.  A point is near (flagged) when it could cross the node box
[0, n - 1] within NEAR E_q (inside: any axis; outside: every axis it lies outside on), |phi| is within NEAR of its E, or the
interpolated g within NEAR of zero.
"""
import contextlib

import numpy as np

import ref64

LEVELSET = 4
_LATTICES = []


def lattice(n, phi):
    """cb200_levelset_prepare in numpy float32: central differences 0.5f * (phi[+1] - phi[-1]) in index units, one-sided on the
    faces; phi flat with i fastest (or indexed [k, j, i])."""
    p = np.asarray(phi, np.float32).reshape(n[2], n[1], n[0])
    out = np.empty(p.shape + (4,), np.float32)
    out[..., 0] = p
    for ch, ax in ((1, 2), (2, 1), (3, 0)):   # g_i along the last axis (i), g_k along the first
        g = np.empty_like(p)
        sl = lambda a, b: tuple(slice(a, b) if d == ax else slice(None) for d in range(3))   # noqa: E731
        g[sl(1, -1)] = np.float32(0.5) * (p[sl(2, None)] - p[sl(None, -2)])
        g[sl(0, 1)] = p[sl(1, 2)] - p[sl(0, 1)]
        g[sl(-1, None)] = p[sl(-1, None)] - p[sl(-2, -1)]
        out[..., ch] = g
    return out


def _cube(lat):
    """each channel as a float64 array indexed [i, j, k], edge-padded to a cube so that ref64's clipped corner reads stay on the
    lattice: (channels[4], M)"""
    ch = np.transpose(np.asarray(lat, np.float64), (3, 2, 1, 0))   # [4, ni, nj, nk]
    M = max(ch.shape[1:])
    pad = [(0, 0)] + [(0, M - s) for s in ch.shape[1:]]
    return np.pad(ch, pad, mode="edge"), M


def levelset_query(o, lat, x):
    """The query of the level-set object o (ref64.object_params: a = node 0, b[0] = c) on the lattice lat (float32[nk, nj, ni, 4])
    at the material-space points x = (value[n, 3], E[n, 3]), as ref64.object_query returns it."""
    nk, nj, ni = lat.shape[:3]
    dims = np.array([ni, nj, nk], np.float64)
    a, c = o["a"], o["b"][0]
    n = len(x[0])
    d = x[0] - a
    q = d / c
    eq = (x[1] + ref64._rnd(d)) / c + ref64._rnd(q)
    viol = (q < 0) | (q > dims - 1)
    inside = ~viol.any(1)
    with np.errstate(divide="ignore", invalid="ignore"):
        m_ax = np.nan_to_num(np.minimum(np.abs(q), np.abs(q - (dims - 1))) / (ref64.EPS32 * eq), nan=np.inf)
    # inside: the nearest face; outside: every violated axis must come in, so the farthest of them
    m_box = np.where(inside, m_ax.min(1), np.where(viol, m_ax, 0.0).max(1))
    i0 = np.clip(np.minimum(np.floor(q), dims - 2), 0, dims - 2).astype(np.int64)
    t = np.clip(q - i0, 0.0, 1.0)
    w = np.stack([1.0 - t, t], -1)
    ew = np.stack([ref64._rnd(1.0 - t), ref64._rnd(t)], -1)
    ch, M = _cube(lat)
    vals = []
    for k in range(4):
        v, e = ref64._trilinear(ch[k], i0, w, ew, M)
        e = e + (ref64._slope(ch[k], i0, w, M, 1.0) * eq).sum(1)
        vals.append((v, e))
    sd, esd = vals[0]
    nr = np.stack([vals[k][0] for k in (1, 2, 3)], 1)
    enr = np.stack([vals[k][1] for k in (1, 2, 3)], 1)
    hit = inside & (sd <= 0)
    m_hit = np.nan_to_num(ref64._margin(sd, esd), nan=np.inf)
    nn = (nr ** 2).sum(1)
    ln = np.sqrt(nn)
    zero = nn == 0
    enr_len = np.sqrt((enr ** 2).sum(1))
    with np.errstate(divide="ignore", invalid="ignore"):
        m_zero = np.where(zero, np.where(enr_len > 0, 0.0, np.inf), ln / (ref64.EPS32 * enr_len))
        on = np.where(zero[:, None], 0.0, nr / np.where(zero, 1.0, ln)[:, None])
        eon = np.where(zero[:, None], 0.0, (2 * enr_len / np.where(zero, 1.0, ln))[:, None] + 3 * np.abs(on))
    margin = np.where(inside, np.minimum(m_box, m_hit), m_box)
    sb = np.where(zero, "levelset_zero", "levelset").astype(object)
    return dict(hit=hit, on=on, eon=eon, zero=zero, m_zero=np.nan_to_num(m_zero, nan=np.inf), margin=margin,
                branch=np.full(n, "miss", dtype=object), shape_branch=np.where(hit, sb, "miss").astype(object))


_object_query = ref64.object_query


def object_query(o, x):
    """ref64.object_query with CB200_SHAPE_LEVELSET answered from the registered lattices"""
    if o["shape"] == LEVELSET:
        return levelset_query(o, _LATTICES[int(o["b"][1])], x)
    return _object_query(o, x)


@contextlib.contextmanager
def registered(lattices):
    """ref64 (object_query and everything that calls it: object_resolve, object_chain, grid_update, substep) with the level-set
    objects' lattices lattices[index]; restored on exit."""
    prev = list(_LATTICES)
    _LATTICES[:] = [np.asarray(l, np.float32) for l in lattices]
    ref64.object_query = object_query
    try:
        yield
    finally:
        ref64.object_query = _object_query
        _LATTICES[:] = prev


def hits(o, lat, t, points):
    """(hit, near) of the world-space float32 points[n, 3] against the level-set object o (a cb200_collision_object) placed at t, as
    cb200_sim_remove_particles tests a particle."""
    p = ref64.object_params(o)
    mp = ref64.material_point(None, p, np.float32(t), points=np.asarray(points, np.float32))
    q = levelset_query(p, np.asarray(lat, np.float32), mp["x"])
    return q["hit"], q["margin"] <= ref64.NEAR
