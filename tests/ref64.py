"""A float64 reference of one sub-step's operations (numpy only, no GPU), with error magnitudes for every output.

Written from the math of MLS-MPM with APIC transfers and from the repository's oracle (oracle/claymore_oracle.c), not
from any other implementation.  It takes the state the engine and the oracle expose between two sub-steps:

* particles per model: rows of ``particle_state`` (x y z, then J for J_FLUID, F column-major for the others, then logJp
  for SAND and NACC);
* material parameters per model: ``params(material, ...)`` below, the float32 values the kernels receive;
* the grid: ``keys`` int[nb, 3] and ``grid`` float[nb, 4, 64] (mass, 3 x momentum; cell x*16 + y*4 + z);
* ``Config`` (domain_bits, boundary, gravity, cfl), ``dt`` and ``new_dt``.

Conventions the engine keeps (DESIGN.md section 3, quirks):
* cell index = round(p / dx), half away from zero; the stencil's base node is cell index - 1; quadratic B-spline;
* #1 the wall mask zeroes a velocity component of a node in a wall band, then gravity is added (also to masked nodes);
* #3 NaN in the max |v|^2 counts as +inf;
* #4 a particle whose new stencil leaves the 8^3 nodes of its particle block's 2x2x2 neighbourhood drops its P2G;
* #6 the fluid's J is clamped at 0.1; #7 FIXED_COROTATED stores the trial F;
* #9 a node whose FP32 mass is subnormal holds no mass for the grid update (the reference flushes subnormals to zero);
* a cell takes at most max_ppc particles at re-bucketing; the rest leave the next partition (``cell_overflow``);
* nodes outside the domain do not exist: what a particle would add there is dropped;
* a signed-distance collider (DESIGN.md section 2.4, C1-C6) acts after the wall mask and gravity on the nodes with mass
  (collider_resolve), then the analytic objects in list order (section 2.9, object_chain); nodes near one of their
  discontinuities, and what reads them, are left out of the checks and counted.

Every output comes with a magnitude M such that an FP32 implementation of the same operations differs from the float64
value by at most a small multiple of 2^-24 * M.  The tests fix that multiple (kappa) per quantity.
"""
import numpy as np

J_FLUID, FIXED_COROTATED, SAND, NACC = 0, 1, 2, 3
CHANNELS = {J_FLUID: 4, FIXED_COROTATED: 12, SAND: 13, NACC: 13}
EPS32 = 2.0 ** -24
FLT_MIN32 = float(np.finfo(np.float32).tiny)   # 2^-126, the smallest normal float32


# ---- parameters ------------------------------------------------------------------------------------------------------
def params(material, rho, vol, *args):
    """Material parameters as the kernels receive them (float32 arithmetic of the update_*_parameters setters).
    FIXED_COROTATED / SAND: (E, nu); J_FLUID: (bulk, gamma, viscosity); NACC: (E, nu, beta, xi)."""
    f = np.float32
    rho, vol = f(rho), f(vol)
    p = dict(material=material, rho=float(rho), volume=float(vol), mass=float(vol * rho),
             bulk=4e4, gamma=7.15, viscosity=0.01, cohesion=0.0, beta=1.0,
             yield_surface=float(f(0.816496580927726) * f(2.0) * f(0.5) / f(2.5)), volume_correction=True,
             xi=0.8, msqr=float(f(3.423772074299613)), hardening_on=True)
    if material == J_FLUID:
        p["bulk"], p["gamma"], p["viscosity"] = (float(f(a)) for a in args)
    else:
        E, nu = f(args[0]), f(args[1])
        lam = E * nu / ((f(1) + nu) * (f(1) - f(2) * nu))
        mu = E / (f(2) * (f(1) + nu))
        p["lambda"], p["mu"] = float(lam), float(mu)
        p["bm"] = float(f(2.0 / 3.0) * mu + lam)
        if material == NACC:
            p["beta"], p["xi"] = float(f(args[2])), float(f(args[3]))
    return p


def scene_params(material, dx):
    """The parameters of the test scenes (claymore_b200.scenes.material_parameters)."""
    vol = dx ** 3 / 8.0
    if material == J_FLUID:
        return params(material, 1e3, vol, 4e4, 7.15, 0.01)
    if material == NACC:
        return params(material, 1e3, vol, 5e3, 0.4, 0.5, 0.8)
    return params(material, 1e3, vol, 5e3, 0.4)


# ---- indices, weights ------------------------------------------------------------------------------------------------
def cell_index(x, dx_inv):
    """round(x / dx), half away from zero."""
    s = np.asarray(x, np.float64) * dx_inv
    return (np.sign(s) * np.floor(np.abs(s) + 0.5)).astype(np.int64)


def bspline(d):
    """Quadratic B-spline weights and their derivatives of a local coordinate d in [0.5, 1.5] (cell units) -> [..., 3]."""
    w = np.stack([0.5 * (1.5 - d) ** 2, 0.75 - (d - 1.0) ** 2, 0.5 * (d - 0.5) ** 2], axis=-1)
    g = np.stack([d - 1.5, -2.0 * (d - 1.0), d - 0.5], axis=-1)
    return w, g


def stencil(pos, dx_inv):
    """base node, local position (cell units), weights W[n,27], weight-gradient magnitudes G[n,27] (cell units) and
    x_i - x_p [n,27,3] (physical units) of particles at pos[n,3]."""
    base = cell_index(pos, dx_inv) - 1
    d = np.asarray(pos, np.float64) * dx_inv - base
    w, g = bspline(d)                                                    # [n,3(axis),3(node)]
    W = (w[:, 0, :, None, None] * w[:, 1, None, :, None] * w[:, 2, None, None, :]).reshape(-1, 27)
    ag = np.abs(g)
    G = (ag[:, 0, :, None, None] * w[:, 1, None, :, None] * w[:, 2, None, None, :]
         + w[:, 0, :, None, None] * ag[:, 1, None, :, None] * w[:, 2, None, None, :]
         + w[:, 0, :, None, None] * w[:, 1, None, :, None] * ag[:, 2, None, None, :]).reshape(-1, 27)
    off = np.stack(np.meshgrid(np.arange(3), np.arange(3), np.arange(3), indexing="ij"), -1).reshape(27, 3)
    xixp = (off[None, :, :] - d[:, None, :]) / dx_inv
    return base, d, W, G, xixp, off


def key_hash(keys):
    keys = np.asarray(keys, np.int64)
    return (keys[..., 0] << 40) | (keys[..., 1] << 20) | keys[..., 2]


class Grid:
    """Keyed grid blocks in float64: ``data[nb, C, 64]``, looked up by node coordinates."""

    def __init__(self, keys, data):
        self.keys = np.asarray(keys, np.int64)
        self.data = np.asarray(data, np.float64)
        h = key_hash(self.keys)
        self._order = np.argsort(h)
        self._sorted = h[self._order]

    def block_of(self, nodes):
        """block index of each node (-1: no such block)."""
        h = key_hash(nodes >> 2)
        i = np.searchsorted(self._sorted, h).clip(0, len(self._sorted) - 1)
        found = self._sorted[i] == h if len(self._sorted) else np.zeros(h.shape, bool)
        return np.where(found, self._order[i], -1)

    def gather(self, nodes):
        """[..., C] values at nodes[..., 3] (0 where the block does not exist) and the existence mask."""
        b = self.block_of(nodes)
        c = (nodes[..., 0] & 3) * 16 + (nodes[..., 1] & 3) * 4 + (nodes[..., 2] & 3)
        v = self.data[b.clip(0), :, c] if len(self.data) else np.zeros(b.shape + (self.data.shape[1],))
        return np.where((b >= 0)[..., None], v, 0.0), b >= 0


class Accumulator:
    """Scatter of node values into keyed blocks (the P2G target): ``add(nodes, values[..., C])``, ``result()``."""

    def __init__(self, nch):
        self.nch = nch
        self.nodes, self.vals = [], []

    def add(self, nodes, vals, keep):
        self.nodes.append(nodes[keep])
        self.vals.append(vals[keep])

    def result(self):
        if not self.nodes:
            return np.zeros((0, 3), np.int64), np.zeros((0, self.nch, 64))
        nodes, vals = np.concatenate(self.nodes), np.concatenate(self.vals)
        h = key_hash(nodes >> 2)
        uh, inv = np.unique(h, return_inverse=True)
        c = (nodes[:, 0] & 3) * 16 + (nodes[:, 1] & 3) * 4 + (nodes[:, 2] & 3)
        out = np.zeros((len(uh), 64, self.nch))
        np.add.at(out, (inv, c), vals)
        keys = np.stack([uh >> 40, (uh >> 20) & 0xFFFFF, uh & 0xFFFFF], -1)
        return keys, out.transpose(0, 2, 1)


def in_domain_nodes(cfg, nodes):
    n = 1 << cfg.domain_bits
    return np.all((nodes >= 0) & (nodes < n), axis=-1)


# ---- rasterize -------------------------------------------------------------------------------------------------------
def rasterize(cfg, models):
    """Initial mass and momentum of ``models`` = [dict(pos[n,3], v0(3), mass)] -> keys, grid[nb,4,64], magnitudes[nb,4,64]."""
    dx_inv = float(1 << cfg.domain_bits)
    acc = Accumulator(8)
    for m in models:
        pos = np.asarray(m["pos"], np.float64)
        base, _, W, _, _, off = stencil(pos, dx_inv)
        nodes = base[:, None, :] + off[None]
        mw = m["mass"] * W
        v0 = np.asarray(m["v0"], np.float64)
        vals = np.concatenate([mw[..., None], mw[..., None] * v0, mw[..., None], mw[..., None] * np.abs(v0)], -1)
        acc.add(nodes, vals, in_domain_nodes(cfg, nodes))
    keys, g = acc.result()
    return keys, g[:, :4], g[:, 4:]


# ---- grid update -----------------------------------------------------------------------------------------------------
def compute_dt(cfg, max_vsq, dt_default, time_left=np.inf):
    """The next dt from the max |v|^2: min(dt_default, dx * cfl / |v|max, time_left) (float64)."""
    dt = float(dt_default)
    mv = np.sqrt(max_vsq)
    if mv > 0:
        dt = min(dt, (1.0 / (1 << cfg.domain_bits)) * float(np.float32(cfg.cfl)) / mv)
    return min(dt, time_left)


def grid_update(cfg, keys, grid, dt, collider=None, t=0.0, objects=None):
    """v = mv / m, wall mask on both faces (key < boundary or key >= G - boundary), then gravity, on the nodes whose mass
    is at least FLT_MIN (a subnormal FP32 mass is no mass: the reference flushes subnormals to zero); other nodes keep
    their momentum channels as they are (0 where nothing was added).  With ``collider`` = (col, sdf, grad) the nodes with
    mass then resolve against it, placed at time ``t`` (collider_resolve), and the max is |v|^2 after the collider (C2).
    Returns (vel[nb,3,64], magnitude[nb,3,64], max |v|^2 over the nodes with mass, NaN -> +inf), and with a collider a
    fourth item: dict(near[nb,64], branch[nb,64], margin[nb,64], vo[nb,3,64], mx_lo, mx_hi, mx_err), the max over every
    choice of the near nodes' branches lying in [mx_lo, mx_hi], and each other node's |v|^2 within kappa 2^-24 mx_err.
    ``objects`` (a non-empty list of cb200_collision_object or object_params) resolve after the collider, in list order
    (object_chain); the info then also holds shape_branch[nb,64] and per list entry its labels (stages)."""
    keys = np.asarray(keys, np.int64)
    grid = np.asarray(grid, np.float64)
    G, bc = 1 << (cfg.domain_bits - 2), cfg.boundary
    wall = (keys < bc) | (keys >= G - bc)                       # [nb, 3]
    m = grid[:, 0]
    has = m >= FLT_MIN32
    with np.errstate(divide="ignore", invalid="ignore"):
        v = grid[:, 1:] / np.where(has, m, 1.0)[:, None]
    v = np.where(has[:, None], np.where(wall[:, :, None], 0.0, v), grid[:, 1:])
    mag = np.abs(v)
    gdt = float(np.float32(cfg.gravity)) * dt
    v[:, 1] += np.where(has, gdt, 0.0)
    mag[:, 1] += np.where(has, abs(gdt), 0.0)
    info = None
    objects = [object_params(o) for o in objects] if objects else []
    if collider is not None or objects:
        nb = len(keys)
        info = dict(near=np.zeros((nb, 64), bool), branch=np.full((nb, 64), "", dtype=object), margin=np.full((nb, 64), np.inf),
                    vo=np.zeros((nb, 3, 64)))
        b, c = np.nonzero(has)
        nodes = keys[b] * 4 + _CELLS[c]
        if objects:
            r = object_chain(cfg, collider, objects, t, nodes, v[b, :, c], mag[b, :, c])
            info["shape_branch"] = np.full((nb, 64), "", dtype=object)
            info["shape_branch"][b, c] = r["shape_branch"]
            info["stages"] = []
            for lab in r["labels"]:
                st = {k: np.full((nb, 64), "" if k.endswith("branch") else False, dtype=object if k.endswith("branch") else bool) for k in lab}
                for k in lab:
                    st[k][b, c] = lab[k]
                info["stages"].append(st)
        else:
            col, sdf, grad = collider
            r = collider_resolve(cfg, col, sdf, grad, t, nodes, v[b, :, c], mag[b, :, c])
        v[b, :, c], mag[b, :, c] = r["v"], r["mag"]
        # g2p2g reads mag as each velocity's scale (the magnitude M of its own roundings), and a velocity resolved exactly
        # (E = 0: the object velocity of a translating static frame, an axis-aligned normal) still has its size.  On the
        # collider path mag stays E, so its g2p2g bound is the tighter one there (too tight, never too loose: with the same
        # floor moving_floor_frame_end's worst F falls from 1.14 to 0.79 of KAPPA); it is kept so that the collider tests'
        # recorded ratios stay comparable.  The objects path, whose exact branches are common, takes the floor.
        if objects:
            mag[b, :, c] = np.maximum(r["mag"], np.abs(r["v"]))
        for f in ("near", "branch", "margin"):
            info[f][b, c] = r[f]
        info["vo"][b, :, c] = r["vo"]
        lo, hi = np.zeros((nb, 64)), np.zeros((nb, 64))
        lo[b, c], hi[b, c] = r["vsq_lo"], r["vsq_hi"]
        info["mx_lo"] = float(np.nan_to_num(lo, nan=np.inf).max(initial=0.0))
        info["mx_hi"] = float(np.nan_to_num(hi, nan=np.inf).max(initial=0.0))
        # E of each resolved node's |v|^2 (sum 2 |v_d| E_d, first order): at a box's edge it can exceed |v|^2 by far
        info["mx_err"] = float(np.where(r["near"], 0.0, (2 * np.abs(r["v"]) * r["mag"]).sum(1)).max(initial=0.0))
    vsq = np.where(has, (v ** 2).sum(1), 0.0)
    vsq = np.where(np.isnan(vsq), np.inf, vsq)
    mx = float(vsq.max()) if vsq.size else 0.0
    return (v, mag, mx) if info is None else (v, mag, mx, info)


# ---- signed-distance collider (DESIGN.md section 2.4, oracle/collider_oracle.c) ----------------------------------------
# Every FP32 quantity of the collider is carried as (value, E): its float64 value and an error magnitude E such that the FP32
# value differs from it by at most a small multiple of 2^-24 * E (first order).  Rules, for exact float32 inputs (E = 0):
#   a + b: Ea + Eb + rnd(a + b);  a * b: Ea |b| + |a| Eb + rnd(a b);  a / b: Ea / |b| + |a| Eb / b^2 + rnd(a / b);
#   sqrt(a): Ea / (2 sqrt a) + rnd(sqrt a);  rnd(r) = |r| unless r is a float32 value (then the operation is exact);
#   sin / cos of an angle a: SINCOS_ULPS |value| + |cos / sin| Ea (the device's sinf / cosf are within a few ulp);
#   trilinear phi (distance or a gradient component) at the material-space point x: sum_c (E_w,c |f_c| + 2 w_c |f_c|) over
#   the 8 corners, plus its sensitivity to the rounding of x, sum_d |d phi / d x_d| E_x,d with |d phi / d x_d| the largest
#   one-sided slope of the cell and of its two neighbours along d (the 1/dx amplification at a box's edges);
#   normalisation: |dn| <= 2 |dn_raw| / |n_raw|, plus the roundings of the sqrt and the division;
#   friction: v += v / len * (vn f) as the products and sums it is, with |vn f| / len taken at most 1 for a positive friction
#   (the slide side at the stick switch, where both sides are 0); a negative friction never sticks and pushes v by more than
#   len where |vn f| > len.
# Exact zeros and exact copies (STICKY's v = 0, the identity frame of a static collider) carry E = 0, so a node of a static
# collider on the lattice is not near the wall band edge it sits on.
# Discontinuities: the hit test (sd <= 0), the wall band (x < lo, x >= hi), the top guard (node gc + 1 >= 4G) and the exact
# zero-normal test.  A node whose distance to one of them is within NEAR x 2^-24 x its own E is "near": its branch may differ
# in FP32, it leaves the checks and is counted.  The approach / separate switch (vn = 0) and the stick / slide switch
# (-vn f = len) are continuous; within NEAR x their error, E is the larger of the two sides'.
STICKY, SLIP, SEPARATE = 0, 1, 2
NEAR = 16.0
SINCOS_ULPS = 4.0
_CELLS = np.stack(np.meshgrid(np.arange(4), np.arange(4), np.arange(4), indexing="ij"), -1).reshape(64, 3)


def _rnd(r):
    r = np.asarray(r, np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        return np.where(np.float32(r).astype(np.float64) == r, 0.0, np.abs(r))


def _add(a, b):
    v = a[0] + b[0]
    return v, a[1] + b[1] + _rnd(v)


def _sub(a, b):
    v = a[0] - b[0]
    return v, a[1] + b[1] + _rnd(v)


def _mul(a, b):
    v = a[0] * b[0]
    return v, a[1] * np.abs(b[0]) + np.abs(a[0]) * b[1] + _rnd(v)


def _div(a, b):
    v = a[0] / b[0]
    return v, a[1] / np.abs(b[0]) + np.abs(a[0]) * b[1] / b[0] ** 2 + _rnd(v)


def _exact(x):
    x = np.asarray(x, np.float64)
    return x, np.zeros_like(x)


def _dot3(a, b, i, j):
    """sum_k a[i(k)] * b[j(k)], k = 0, 1, 2 left to right (a, b: (value, E) with the components on the last axis)."""
    s = None
    for k in range(3):
        p = _mul((a[0][..., i(k)], a[1][..., i(k)]), (b[0][..., j(k)], b[1][..., j(k)]))
        s = p if s is None else _add(s, p)
    return s


def collider_params(c):
    """The collider's float32 parameters as float64 values: a cb200_collider / orc_collider struct or a dict with its fields."""
    get = (lambda k: c[k]) if isinstance(c, dict) else (lambda k: getattr(c, k))
    f = lambda x: np.asarray(np.asarray(x, np.float32), np.float64)   # noqa: E731
    return dict(rot_mat=f(list(get("rot_mat"))).reshape(9), trans=f(list(get("trans"))), trans_vel=f(list(get("trans_vel"))),
                omega=f(list(get("omega"))), dsdt=float(f(get("dsdt"))), scale=float(f(get("scale"))), friction=float(f(get("friction"))),
                type=int(get("type")))


def collider_frame(col, t):
    """The collider's frame at the float32 time t: rot (9, storage (i, j) at 3i + j) = Rz(w_z t) Ry(w_y t) Rx(w_x t) rot_mat in
    storage order (collider_mat_mul multiplies the new axis rotation from the left), b = trans + trans_vel t,
    s_inv = 1 / (1 + dsdt t); each as (value, E)."""
    col = collider_params(col)
    t = float(np.float32(t))
    cur = _exact(col["rot_mat"])
    for d in range(3):
        a = _mul(_exact(col["omega"][d]), _exact(t))
        c, s = np.cos(a[0]), np.sin(a[0])
        ec, es = SINCOS_ULPS * abs(c) + abs(s) * a[1], SINCOS_ULPS * abs(s) + abs(c) * a[1]
        if a[0] == 0.0:
            c, s, ec, es = 1.0, 0.0, 0.0, 0.0                     # sinf(0) = 0, cosf(0) = 1 exactly
        r, er = np.zeros(9), np.zeros(9)
        one = [0, 4, 8][d]
        r[one] = 1.0
        ci, si, mi = {0: ((4, 8), 7, 5), 1: ((0, 8), 2, 6), 2: ((0, 4), 3, 1)}[d]
        r[list(ci)], er[list(ci)] = c, ec
        r[si], er[si] = s, es
        r[mi], er[mi] = -s, es
        # c[3j + i] = a[i] b[3j] + a[3 + i] b[3j + 1] + a[6 + i] b[3j + 2], a = the previous frame, b = the axis rotation
        nv, ne = np.zeros(9), np.zeros(9)
        for j in range(3):
            for i in range(3):
                v = _dot3(cur, (r, er), lambda k, i=i: 3 * k + i, lambda k, j=j: 3 * j + k)
                nv[3 * j + i], ne[3 * j + i] = v
        cur = (nv, ne)
    b = _add(_exact(col["trans"]), _mul(_exact(col["trans_vel"]), _exact(t)))
    s_inv = _div(_exact(1.0), _add(_exact(1.0), _mul(_exact(col["dsdt"]), _exact(t))))
    return dict(rot=cur, b=b, s_inv=s_inv, t=t, col=col)


def _trilinear(f, gc, w, ew, N):
    """phi at the 8 corners gc + {0, 1}^3 of the dense field f[(N, N, N)] with weights w[n, 3, 2] (errors ew), and its E
    without the position sensitivity."""
    val, err = 0.0, 0.0
    for i in range(2):
        for j in range(2):
            for k in range(2):
                fc = f[np.minimum(gc[:, 0] + i, N - 1), np.minimum(gc[:, 1] + j, N - 1), np.minimum(gc[:, 2] + k, N - 1)].astype(np.float64)
                wc = w[:, 0, i] * w[:, 1, j] * w[:, 2, k]
                ewc = ew[:, 0, i] * w[:, 1, j] * w[:, 2, k] + w[:, 0, i] * ew[:, 1, j] * w[:, 2, k] + w[:, 0, i] * w[:, 1, j] * ew[:, 2, k]
                val = val + wc * fc
                err = err + ewc * np.abs(fc) + 2 * wc * np.abs(fc)
    return val, err


def _slope(f, gc, w, N, dx):
    """[n, 3]: the largest |d phi / d x_d| of the trilinear interpolant over the cell gc and its two neighbours along d."""
    out = np.zeros((len(gc), 3))
    for d in range(3):
        o1, o2 = [e for e in range(3) if e != d]
        for shift in (-1, 0, 1):
            s = 0.0
            for i in range(2):
                for j in range(2):
                    idx_lo, idx_hi = [None] * 3, [None] * 3
                    idx_lo[o1] = idx_hi[o1] = np.clip(gc[:, o1] + i, 0, N - 1)
                    idx_lo[o2] = idx_hi[o2] = np.clip(gc[:, o2] + j, 0, N - 1)
                    idx_lo[d] = np.clip(gc[:, d] + shift, 0, N - 1)
                    idx_hi[d] = np.clip(gc[:, d] + shift + 1, 0, N - 1)
                    s = s + w[:, o1, i] * w[:, o2, j] * (f[tuple(idx_hi)].astype(np.float64) - f[tuple(idx_lo)])
            out[:, d] = np.maximum(out[:, d], np.abs(s) / dx)
    return out


def material_point(cfg, col, t, nodes):
    """The collider's (or an object's) frame at the float32 time t and the material-space point of each node nodes[n, 3]:
    dict(f (collider_frame), col (collider_params), Rb (the rotation per node, (value, E)), xm (node dx - b), x (the
    material-space point R (node dx - b) s_inv scale + trans)), every vector as (value[n, 3], E[n, 3])."""
    f = collider_frame(col, t)
    col = f["col"]
    nodes = np.asarray(nodes, np.int64).reshape(-1, 3)
    n = len(nodes)
    dx = 1.0 / (1 << cfg.domain_bits)
    R = f["rot"]
    Rb = (np.broadcast_to(R[0], (n, 9)), np.broadcast_to(R[1], (n, 9)))
    xm = _sub(_exact(nodes * dx), (np.broadcast_to(f["b"][0], (n, 3)), np.broadcast_to(f["b"][1], (n, 3))))
    x0 = _mul(xm, f["s_inv"])
    y = [_dot3(Rb, x0, lambda k, d=d: 3 * d + k, lambda k: k) for d in range(3)]
    y = (np.stack([a[0] for a in y], -1), np.stack([a[1] for a in y], -1))
    x = _add(_mul(y, _exact(col["scale"])), _exact(col["trans"]))
    return dict(f=f, col=col, Rb=Rb, xm=xm, x=x)


def levelset_query(cfg, sdf, grad, x):
    """collider_query of the dense level set sdf[(N, N, N)], grad[(3, N, N, N)] (read by node index) at the material-space
    points x = (value[n, 3], E[n, 3]).  Returns the query dict collider_resolve takes: hit, on / eon (the material-space
    normal and its E), zero (no normal), m_zero (its margin), margin (of the wall band, the top guard and the hit test),
    branch (the label of a node that is not hit)."""
    n = len(x[0])
    G = 1 << (cfg.domain_bits - 2)
    N, bc = 4 * G, cfg.boundary
    dx = 1.0 / (1 << cfg.domain_bits)
    # wall band, top guard, trilinear distance and gradient
    lo, hi = float(bc) * dx * 4.0, float(G - bc) * 4.0 * dx
    band = np.any((x[0] < lo) | (x[0] >= hi), axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        m_band = np.min(np.minimum(np.abs(x[0] - lo), np.abs(x[0] - hi)) / (EPS32 * x[1]), axis=1)
    gc = np.clip(np.floor(x[0] / dx), 0, N - 1).astype(np.int64)
    top = ~band & np.any(gc + 1 >= N, axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        m_top = np.min(np.abs(x[0] - (N - 1) * dx) / (EPS32 * x[1]), axis=1)
    gcs = np.minimum(gc, N - 2)
    dl = x[0] - gcs * dx
    w = np.stack([1.0 - dl / dx, dl / dx], -1)                                 # [n, 3, 2]
    ew = np.stack([_rnd(1.0 - dl / dx), _rnd(dl / dx)], -1)                    # the rounding of 1 - dl / dx (dl / dx is exact)
    sd, esd = _trilinear(sdf, gcs, w, ew, N)
    esd = esd + (_slope(sdf, gcs, w, N, dx) * x[1]).sum(1)                     # the sensitivity to the rounding of x
    nr, enr = np.zeros((n, 3)), np.zeros((n, 3))
    for d in range(3):
        nr[:, d], enr[:, d] = _trilinear(grad[d], gcs, w, ew, N)
        enr[:, d] += (_slope(grad[d], gcs, w, N, dx) * x[1]).sum(1)
    hit = ~band & ~top & (sd <= 0)
    with np.errstate(divide="ignore", invalid="ignore"):
        m_hit = np.abs(sd) / (EPS32 * esd)
    nn = (nr ** 2).sum(1)
    ln = np.sqrt(nn)
    zero = nn == 0
    enr_len = np.sqrt((enr ** 2).sum(1))
    with np.errstate(divide="ignore", invalid="ignore"):
        m_zero = np.where(zero, np.where(enr_len > 0, 0.0, np.inf), ln / (EPS32 * enr_len))
        on = np.where(zero[:, None], 0.0, nr / np.where(zero, 1.0, ln)[:, None])
        eon = np.where(zero[:, None], 0.0, (2 * enr_len / np.where(zero, 1.0, ln))[:, None] + 3 * np.abs(on))
    branch = np.where(band, "band", np.where(top, "top", "miss")).astype(object)
    margin = np.where(band | top, np.minimum(m_band, m_top), np.minimum(np.minimum(m_band, m_top), m_hit))
    return dict(hit=hit, on=on, eon=eon, zero=zero, m_zero=m_zero, margin=margin, branch=branch)


def collider_resolve(cfg, col, sdf, grad, t, nodes, v, vmag):
    """detect_and_resolve_collision of the velocities v[n, 3] (magnitudes vmag[n, 3]) at the grid nodes nodes[n, 3], the
    collider col (collider_params) placed at the float32 time t, its level set the dense sdf[(N, N, N)], grad[(3, N, N, N)]
    read by node index.  Returns dict(v, mag (E of each component), vo (the object velocity), hit, branch (label), margin
    (distance to the nearest discontinuity in units of 2^-24 E), near, vsq_lo, vsq_hi (|v|^2 over both sides of a near
    node's branch)) and what object_chain needs to follow a near node's branches."""
    p = material_point(cfg, col, t, nodes)
    return resolve_query(p, levelset_query(cfg, sdf, grad, p["x"]), v, vmag)


def resolve_query(p, q, v, vmag):
    """The object velocity and the response of the collider or object p["col"] (material_point p) to the query q at the nodes
    with velocities v[n, 3] (magnitudes vmag[n, 3]), shared by the level set and the analytic shapes (collider_resolve)."""
    col, Rb, xm, x = p["col"], p["Rb"], p["xm"], p["x"]
    n = len(xm[0])
    vin = (np.asarray(v, np.float64).reshape(n, 3), np.asarray(vmag, np.float64).reshape(n, 3))
    tol = EPS32 * NEAR
    hit, on, eon, zero, m_zero = q["hit"], q["on"], q["eon"], q["zero"], q["m_zero"]
    # object velocity: omega x xm + xm dsdt / scale + R^T (omega (all-plus) r + trans_vel) scale + trans_vel, r = x - trans
    wv = _exact(np.broadcast_to(col["omega"], (n, 3)))
    cross = [_sub(_mul((wv[0][:, a], wv[1][:, a]), (xm[0][:, b], xm[1][:, b])), _mul((wv[0][:, b], wv[1][:, b]), (xm[0][:, a], xm[1][:, a])))
             for a, b in ((1, 2), (2, 0), (0, 1))]
    vo = (np.stack([c[0] for c in cross], -1), np.stack([c[1] for c in cross], -1))
    ds = _div(_exact(col["dsdt"]), _exact(col["scale"]))
    vo = _add(vo, _mul(xm, ds))
    r = _sub(x, _exact(col["trans"]))
    tv = _exact(np.broadcast_to(col["trans_vel"], (n, 3)))
    mv = [_add(_add(_mul((wv[0][:, a], wv[1][:, a]), (r[0][:, b], r[1][:, b])), _mul((wv[0][:, b], wv[1][:, b]), (r[0][:, a], r[1][:, a]))),
               (tv[0][:, d], tv[1][:, d])) for d, (a, b) in enumerate(((1, 2), (2, 0), (0, 1)))]
    mv = (np.stack([m[0] for m in mv], -1), np.stack([m[1] for m in mv], -1))
    rot_t = [_dot3(Rb, mv, lambda k, d=d: d + 3 * k, lambda k: k) for d in range(3)]
    rot_t = (np.stack([a[0] for a in rot_t], -1), np.stack([a[1] for a in rot_t], -1))
    vo = _add(vo, _add(_mul(rot_t, _exact(col["scale"])), tv))
    # resolve
    vr = _sub(vin, vo)
    typ, fr = col["type"], col["friction"]
    out_v, out_e = vin[0].copy(), vin[1].copy()
    branch = q["branch"].copy()
    margin = q["margin"]
    m_hit = np.nan_to_num(margin, nan=np.inf)                               # the hit test's: a near node may miss or hit
    zero_alt = np.zeros(n, bool)
    res_v, res_e = vo[0].copy(), vo[1].copy()                               # STICKY: v = 0 + vo
    if typ == STICKY:
        lab = np.full(n, "sticky", dtype=object)
    else:
        nv = [_dot3(Rb, (on, eon), lambda k, d=d: d + 3 * k, lambda k: k) for d in range(3)]
        nvec = (np.stack([a[0] for a in nv], -1), np.stack([a[1] for a in nv], -1))
        vn = _dot3(nvec, vr, lambda k: k, lambda k: k)
        proj = _sub(vr, _mul(nvec, (vn[0][:, None], vn[1][:, None])))
        fric = (fr > 0) if typ == SLIP else (fr != 0)
        ln2 = (proj[0] ** 2).sum(1)
        plen = np.sqrt(ln2)
        eplen = np.where(plen > 0, (np.abs(proj[0]) * proj[1]).sum(1) / np.where(plen > 0, plen, 1.0), np.sqrt((proj[1] ** 2).sum(1))) + _rnd(plen)
        vnf = _mul(vn, _exact(fr))
        with np.errstate(divide="ignore", invalid="ignore"):
            qf = np.abs(vnf[0]) / plen                                  # a negative friction has no stick side: |vn f| / len may exceed 1
            qf = np.where(plen > 0, np.minimum(qf, 1.0) if fr > 0 else qf, 1.0)
            unit = proj[0] / np.where(plen > 0, plen, 1.0)[:, None]
        slide_v = proj[0] + unit * vnf[0][:, None]
        slide_e = proj[1] * (1 + qf)[:, None] + np.abs(unit) * (vnf[1] + qf * eplen)[:, None] + _rnd(slide_v)
        stick = -vnf[0] >= plen
        with np.errstate(divide="ignore", invalid="ignore"):
            near_stick = np.abs(plen + vnf[0]) <= tol * (eplen + vnf[1])
            near_vn = np.abs(vn[0]) <= tol * vn[1]
        approach = vn[0] < 0
        use_fric = fric & approach
        fv = np.where(use_fric[:, None], np.where(stick[:, None], 0.0, slide_v), proj[0])
        fe = np.where(use_fric[:, None], np.where(stick[:, None] & ~near_stick[:, None], 0.0, slide_e), proj[1])
        fe = np.where((fric & near_vn)[:, None], np.maximum(fe, np.maximum(slide_e, proj[1])), fe)
        if typ == SLIP:
            sv, se = fv, fe
            lab = np.where(use_fric, np.where(stick, "slip_stick", "slip_friction"), "slip").astype(object)
        else:
            sv = np.where(approach[:, None], fv, vr[0])
            se = np.where(approach[:, None], fe, vr[1])
            se = np.where(near_vn[:, None], np.maximum(se, np.maximum(fe, vr[1])), se)
            lab = np.where(approach, "separate_approach", "separate_separate").astype(object)
        res_v, res_e = _add((sv, se), vo)
        # zero normal (C5): SEPARATE gives 0 (it returns before the object velocity is added back); SLIP's projection on n = 0
        # leaves v - vo as it is, and adding vo back gives v up to the two roundings the general path already carries
        if typ == SEPARATE:
            res_v = np.where(zero[:, None], 0.0, res_v)
            res_e = np.where(zero[:, None], 0.0, res_e)
        lab = np.where(zero, "zero_normal", lab)
        margin = np.where(hit, np.minimum(margin, m_zero), margin)
        zero_alt = hit & (np.nan_to_num(m_zero, nan=np.inf) <= NEAR)
    out_v = np.where(hit[:, None], res_v, out_v)
    out_e = np.where(hit[:, None], res_e, out_e)
    branch = np.where(hit, lab, branch)
    margin = np.nan_to_num(margin, nan=np.inf)            # 0 / 0: an exact quantity on the discontinuity, decided alike
    near = margin <= NEAR
    # |v|^2 over both sides of a near node: hit <-> no hit, and for a near zero normal any unit normal
    vsq = (out_v ** 2).sum(1)
    alt_hit = (res_v ** 2).sum(1)
    alt_miss = (vin[0] ** 2).sum(1)
    lo_sq = np.where(near, np.minimum(alt_hit, alt_miss), vsq)
    hi_sq = np.where(near, np.maximum(alt_hit, alt_miss), vsq)
    span = np.zeros(n)
    ovo = np.sqrt((vo[0] ** 2).sum(1))
    if typ != STICKY:
        span = (1 + abs(fr)) * np.sqrt((vr[0] ** 2).sum(1))
        lo_sq = np.where(zero_alt, np.minimum(lo_sq, np.maximum(ovo - span, 0.0) ** 2), lo_sq)
        hi_sq = np.where(zero_alt, np.maximum(hi_sq, (ovo + span) ** 2), hi_sq)
    return dict(v=out_v, mag=out_e, vo=vo[0], hit=hit, branch=branch, margin=margin, near=near, vsq_lo=lo_sq, vsq_hi=hi_sq,
                res_v=res_v, near_hit=m_hit <= NEAR, normal_alt=zero_alt, ovo=ovo, span=span, shape_branch=q.get("shape_branch"),
                type=typ, friction=fr)


# ---- analytic collision objects (DESIGN.md section 2.9, object_query in collider.cuh) ------------------------------------
# The object's frame, material-space point, object velocity and response are the collider's (material_point, resolve_query);
# only the query differs.  Each query's quantities carry E by the rules above, plus sqrt(a) near 0: at most sqrt(Ea / 2^-24)
# in units of 2^-24 (|sqrt(a + e) - sqrt(a)| <= sqrt(|e|)).  Discontinuities and their margins (distance / (2^-24 E)):
#   plane  phi = (x - a) . b <= 0, b the stored unit normal (exact);
#   box    the six comparisons a_d <= x_d <= b_d (a miss flips only if every failing one does: its margin is their largest),
#          the axis of the largest q_d = max(a_d - x_d, x_d - b_d) (a strict > : the lowest axis wins a tie), and the face's
#          sign ql > qh (+1 at the exact centre);
#   sphere dd = |x - a|^2 <= r * r (with the rounding of r * r), the zero-normal test dd > 0, n = d / sqrt(dd);
#   cylinder rho2 = d0^2 + d2^2 <= r * r and |d1| <= h, the cap / side switch h - |d1| < r - rho, the cap's sign d1 < 0, the
#          side's zero-normal test rho > 0, n = (d0, 0, d2) / rho.
# An exact quantity exactly on a switch (E = 0: 0 / 0) is decided alike, as above.  A hit node near a normal switch (box axis
# or sign, cylinder cap or side, a zero normal) may take any unit normal in FP32: object_chain bounds it by the span bound.
PLANE, BOX, SPHERE, CYLINDER = 0, 1, 2, 3
MAX_CANDIDATES = 8     # object_chain: a node's branch candidates beyond this many collapse into one speed interval


def object_params(o):
    """An object's float32 fields as float64 values (a cb200_collision_object or a dict with its fields), the plane normal as
    cb200_sim_set_collision_objects stores it: made unit length in double once more and rounded to float32."""
    get = (lambda k: o[k]) if isinstance(o, dict) else (lambda k: getattr(o, k))
    p = collider_params(o)
    f32 = lambda x: np.asarray(np.asarray(x, np.float32), np.float64)   # noqa: E731
    p.update(shape=int(get("shape")), a=f32(list(get("a"))), b=f32(list(get("b"))))
    if p["shape"] == PLANE:
        p["b"] = f32(p["b"] / np.sqrt((p["b"] * p["b"]).sum()))
    return p


def _col(x, k):
    return x[0][:, k], x[1][:, k]


def _margin(dist, err):
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.abs(dist) / (EPS32 * err)


def _sqrt(a):
    v = np.sqrt(a[0])
    with np.errstate(divide="ignore", invalid="ignore"):
        flat = np.sqrt(a[1] / EPS32)
        e = np.where(v > 0, np.minimum(a[1] / (2 * np.where(v > 0, v, 1.0)), flat), flat)
    return v, e + _rnd(v)


def _both(conds, margins):
    """hit = every condition, and its margin: the smallest over all when it holds, else the largest over the failing ones."""
    conds, margins = np.stack(conds, 1), np.nan_to_num(np.stack(margins, 1), nan=np.inf)
    hit = conds.all(1)
    return hit, np.where(hit, margins.min(1), np.where(conds, 0.0, margins).max(1))


def object_query(o, x):
    """object_query of the object o (object_params) at the material-space points x = (value[n, 3], E[n, 3]): the query dict of
    resolve_query (the normal margins folded into m_zero, so that a node near any normal switch is near and bounded by
    the span bound), plus shape_branch (the shape's branch label of each hit node)."""
    n = len(x[0])
    a, b, shape = o["a"], o["b"], o["shape"]
    on, eon = np.zeros((n, 3)), np.zeros((n, 3))
    zero = np.zeros(n, bool)
    m_norm = np.full(n, np.inf)
    d = [_sub(_col(x, k), _exact(a[k])) for k in range(3)]
    if shape == PLANE:
        phi = _add(_add(_mul(d[0], _exact(b[0])), _mul(d[1], _exact(b[1]))), _mul(d[2], _exact(b[2])))
        hit, margin = phi[0] <= 0, _margin(phi[0], phi[1])
        on[:] = b
        sb = np.full(n, "plane", dtype=object)
    elif shape == BOX:
        conds, ms = [], []
        for k in range(3):
            conds += [a[k] <= x[0][:, k], x[0][:, k] <= b[k]]
            ms += [_margin(x[0][:, k] - a[k], x[1][:, k]), _margin(x[0][:, k] - b[k], x[1][:, k])]
        hit, margin = _both(conds, ms)
        ql = [_sub(_exact(a[k]), _col(x, k)) for k in range(3)]
        qh = [_sub(_col(x, k), _exact(b[k])) for k in range(3)]
        qv = np.stack([np.maximum(ql[k][0], qh[k][0]) for k in range(3)], 1)
        qe = np.stack([np.maximum(ql[k][1], qh[k][1]) for k in range(3)], 1)
        axis = np.argmax(qv, 1)                                             # the first of equal maxima: the lowest axis
        i = np.arange(n)
        for k in range(3):
            m_ax = np.nan_to_num(_margin(qv[i, axis] - qv[:, k], qe[i, axis] + qe[:, k]), nan=np.inf)
            m_norm = np.minimum(m_norm, np.where(axis == k, np.inf, m_ax))
        qlv = np.stack([c[0] for c in ql], 1)[i, axis]
        qhv = np.stack([c[0] for c in qh], 1)[i, axis]
        sgn = np.where(qlv > qhv, -1.0, 1.0)
        m_sgn = _margin(qlv - qhv, np.stack([c[1] for c in ql], 1)[i, axis] + np.stack([c[1] for c in qh], 1)[i, axis])
        m_norm = np.minimum(m_norm, np.nan_to_num(m_sgn, nan=np.inf))
        on[i, axis] = sgn
        sb = np.array([f"box_{'xyz'[k]}{'-' if s < 0 else '+'}" for k, s in zip(axis, sgn)], dtype=object)
    elif shape == SPHERE:
        dd = _add(_add(_mul(d[0], d[0]), _mul(d[1], d[1])), _mul(d[2], d[2]))
        rr = _mul(_exact(b[0]), _exact(b[0]))
        hit, margin = dd[0] <= rr[0], _margin(dd[0] - rr[0], dd[1] + rr[1])
        zero = dd[0] == 0
        m_norm = np.nan_to_num(_margin(dd[0], dd[1]), nan=np.inf)
        ln = _sqrt(dd)
        safe = (np.where(zero, 1.0, ln[0]), ln[1])
        for k in range(3):
            c = _div(d[k], safe)
            on[:, k], eon[:, k] = np.where(zero, 0.0, c[0]), np.where(zero, 0.0, c[1])
        sb = np.where(zero, "sphere_zero", "sphere").astype(object)
    else:
        h = b[1]
        rho2 = _add(_mul(d[0], d[0]), _mul(d[2], d[2]))
        rr = _mul(_exact(b[0]), _exact(b[0]))
        ad1 = (np.abs(d[1][0]), d[1][1])
        hit, margin = _both([rho2[0] <= rr[0], ad1[0] <= h], [_margin(rho2[0] - rr[0], rho2[1] + rr[1]), _margin(ad1[0] - h, ad1[1])])
        rho = _sqrt(rho2)
        A, B = _sub(_exact(h), ad1), _sub(_exact(b[0]), rho)
        cap = A[0] < B[0]
        m_cap = np.nan_to_num(_margin(A[0] - B[0], A[1] + B[1]), nan=np.inf)
        m_csgn = np.nan_to_num(_margin(d[1][0], d[1][1]), nan=np.inf)
        zero = ~cap & (rho[0] == 0)
        m_zero_side = np.nan_to_num(_margin(rho2[0], rho2[1]), nan=np.inf)
        m_norm = np.minimum(m_cap, np.where(cap, m_csgn, m_zero_side))
        on[:, 1] = np.where(cap, np.where(d[1][0] < 0, -1.0, 1.0), 0.0)
        safe = (np.where(rho[0] > 0, rho[0], 1.0), rho[1])
        for k in (0, 2):
            c = _div(d[k], safe)
            side = ~cap & ~zero
            on[:, k], eon[:, k] = np.where(side, c[0], 0.0), np.where(side, c[1], 0.0)
        tie = (A[0] == B[0]) & (A[1] == 0) & (B[1] == 0)                    # an exact cap / side tie: the side wins
        sb = np.where(cap, np.where(d[1][0] < 0, "cyl_cap-", "cyl_cap+"), np.where(zero, "cyl_zero", np.where(tie, "cyl_side_tie", "cyl_side"))).astype(object)
    return dict(hit=hit, on=on, eon=eon, zero=zero, m_zero=m_norm, margin=margin, branch=np.full(n, "miss", dtype=object),
                shape_branch=np.where(hit, sb, "miss").astype(object))


def object_resolve(cfg, o, t, nodes, v, vmag):
    """collider_resolve with the analytic object o (object_params) in place of the level set."""
    p = material_point(cfg, o, t, nodes)
    return resolve_query(p, object_query(o, p["x"]), v, vmag)


def object_chain(cfg, collider, objects, t, nodes, v, vmag):
    """The level-set collider = (col, sdf, grad) (or None), then each object (object_params) in list order, each resolving
    the velocity and E the previous one left, all placed at the float32 time t.  Returns collider_resolve's dict with near
    the union over the list, margin the smallest, branch the last hit's label (shape_branch likewise: labels[i] per stage in
    ``labels``), and vsq_lo / vsq_hi over every branch choice of the near nodes: their candidate velocities are carried
    through the list, each near decision adding the other branch; a near normal switch (any unit normal) and a node with more
    than MAX_CANDIDATES candidates carry a speed interval instead."""
    nodes = np.asarray(nodes, np.int64).reshape(-1, 3)
    stages = []
    if collider is not None:
        col, sdf, grad = collider
        stages.append(lambda nd, vv, vm: collider_resolve(cfg, col, sdf, grad, t, nd, vv, vm))
    for o in objects:
        stages.append(lambda nd, vv, vm, o=o: object_resolve(cfg, o, t, nd, vv, vm))
    n = len(nodes)
    v0 = np.asarray(v, np.float64).reshape(n, 3)
    cur, mag = v0, np.asarray(vmag, np.float64).reshape(n, 3)
    near, margin = np.zeros(n, bool), np.full(n, np.inf)
    branch, shape_branch = np.full(n, "miss", dtype=object), np.full(n, "miss", dtype=object)
    labels, vo = [], np.zeros((n, 3))
    for st in stages:
        r = st(nodes, cur, mag)
        cur, mag = r["v"], r["mag"]
        near |= r["near"]
        margin = np.minimum(margin, r["margin"])
        branch = np.where(r["hit"], r["branch"], branch)
        sb = r["shape_branch"] if r["shape_branch"] is not None else np.where(r["hit"], "levelset", "miss").astype(object)
        shape_branch = np.where(r["hit"], sb, shape_branch)
        vo = np.where(r["hit"][:, None], r["vo"], vo)
        labels.append(dict(hit=r["hit"], near=r["near"], branch=r["branch"], shape_branch=sb))
    vsq = (cur ** 2).sum(1)
    lo, hi = vsq.copy(), vsq.copy()
    S = np.flatnonzero(near)
    if len(S):
        # candidate rows: (owner in S, velocity) or (owner, speed interval [slo, shi]) with a NaN velocity
        own = np.arange(len(S))
        rv = v0[S].copy()
        iv = np.full((len(S), 2), np.nan)
        for st in stages:
            isint = ~np.isnan(iv[:, 0])
            r = st(nodes[S][own], np.where(isint[:, None], 0.0, rv), np.zeros((len(own), 3)))
            sticky, fr = r["type"] == STICKY, abs(r["friction"])
            no, nv, ni = [], [], []
            for j in range(len(own)):
                hit, nh, ovo, span = bool(r["hit"][j]), bool(r["near_hit"][j]), r["ovo"][j], r["span"][j]
                if hit or nh:                                           # the hit branch
                    if sticky:
                        no.append(own[j]), nv.append(r["vo"][j]), ni.append((np.nan, np.nan))
                    elif isint[j]:                                      # |v - vo| <= (1 + |friction|) |v_in - vo|
                        no.append(own[j]), nv.append(np.zeros(3)), ni.append((0.0, ovo + (1 + fr) * (iv[j][1] + ovo)))
                    elif r["normal_alt"][j]:                            # any unit normal (SEPARATE's zero normal: 0)
                        no.append(own[j]), nv.append(np.zeros(3)), ni.append((0.0 if r["type"] == SEPARATE else max(ovo - span, 0.0), ovo + span))
                    else:
                        no.append(own[j]), nv.append(r["res_v"][j]), ni.append((np.nan, np.nan))
                if nh or not hit:                                       # the miss branch: the row as it is
                    no.append(own[j]), nv.append(rv[j]), ni.append(iv[j])
            own, rv, iv = np.asarray(no, np.int64), np.asarray(nv, np.float64).reshape(-1, 3), np.asarray(ni, np.float64).reshape(-1, 2)
            own, rv, iv = _cap_candidates(own, rv, iv)
        sp_lo = np.where(np.isnan(iv[:, 0]), np.sqrt((rv ** 2).sum(1)), iv[:, 0])
        sp_hi = np.where(np.isnan(iv[:, 0]), np.sqrt((rv ** 2).sum(1)), iv[:, 1])
        clo, chi = np.full(len(S), np.inf), np.zeros(len(S))
        np.minimum.at(clo, own, sp_lo ** 2)
        np.maximum.at(chi, own, sp_hi ** 2)
        lo[S], hi[S] = clo, chi
    return dict(v=cur, mag=mag, vo=vo, near=near, margin=margin, branch=branch, shape_branch=shape_branch, labels=labels,
                vsq_lo=lo, vsq_hi=hi)


def _cap_candidates(own, rv, iv):
    """A node with more than MAX_CANDIDATES rows keeps one: the speed interval over them."""
    cnt = np.bincount(own, minlength=own.max(initial=-1) + 1)
    big = cnt[own] > MAX_CANDIDATES
    if not big.any():
        return own, rv, iv
    sp = np.sqrt((rv ** 2).sum(1))
    slo, shi = np.where(np.isnan(iv[:, 0]), sp, iv[:, 0]), np.where(np.isnan(iv[:, 0]), sp, iv[:, 1])
    keep = ~big
    out_o, out_v, out_i = [own[keep]], [rv[keep]], [iv[keep]]
    for o in np.unique(own[big]):
        m = own == o
        out_o.append(np.array([o])), out_v.append(np.zeros((1, 3))), out_i.append(np.array([[slo[m].min(), shi[m].max()]]))
    return np.concatenate(out_o), np.concatenate(out_v), np.concatenate(out_i)


# ---- constitutive models (exact float64) -------------------------------------------------------------------------------
def signed_svd(F):
    """F = U diag(S) V^T with U, V rotations; the sign of det F goes on the smallest singular value."""
    U, S, Vt = np.linalg.svd(F)
    V = np.swapaxes(Vt, -1, -2).copy()
    U = U.copy()
    for M in (U, V):
        neg = np.linalg.det(M) < 0
        M[neg, :, 2] *= -1
        S[neg, 2] *= -1
    return U, S, V


def _udv(U, s, V):
    return np.einsum("nij,nj,nkj->nik", U, s, V)


def stress_fixed_corotated(p, F):
    """P F^T vol = (2 mu (F - R) F^T + lambda (J - 1) J I) vol, R the polar rotation."""
    U, S, V = signed_svd(F)
    R = U @ np.swapaxes(V, -1, -2)
    J = np.prod(S, -1)
    PF = 2 * p["mu"] * (F - R) @ np.swapaxes(F, -1, -2) + (p["lambda"] * (J - 1) * J)[:, None, None] * np.eye(3)
    return PF * p["volume"]


def stress_sand(p, F, log_jp):
    """Drucker-Prager return mapping (Klar et al.) in Hencky strain; returns (F, PF, logJp, margin to a branch point)."""
    mu, lam, coh = p["mu"], p["lambda"], p["cohesion"]
    U, S, V = signed_svd(F)
    eps = np.log(np.maximum(np.abs(S), 1e-4)) - coh
    sum_eps = eps.sum(-1)
    tr = sum_eps + log_jp
    eh = eps - tr[:, None] / 3
    ehn = np.linalg.norm(eh, axis=-1)
    dg = ehn + (3 * lam + 2 * mu) / (2 * mu) * tr * p["yield_surface"]
    tip = tr >= 0
    with np.errstate(divide="ignore", invalid="ignore"):
        H = np.where((dg <= 0)[:, None], eps + coh, eps - (dg / ehn)[:, None] * eh + coh)
    newS = np.where(tip[:, None], np.exp(coh), np.exp(H))
    new_ljp = np.where(tip, p["beta"] * sum_eps + log_jp if p["volume_correction"] else log_jp, 0.0)
    Fn = _udv(U, newS, V)
    ls = np.log(newS)
    Ph = (2 * mu * ls + lam * ls.sum(-1, keepdims=True)) / newS
    PF = _udv(U, Ph, V) @ np.swapaxes(Fn, -1, -2) * p["volume"]
    margin = np.where(tip, np.abs(tr), np.minimum(np.abs(tr), np.abs(dg)))
    branch = np.where(tip, "tip", np.where(dg <= 0, "elastic", "yield"))
    return Fn, PF, new_ljp, margin, branch


def stress_nacc(p, F, log_jp):
    """Non-associated Cam-clay (Wolper et al. 2019) with hardening; returns (F, PF, logJp, margin to a branch point)."""
    mu, bm, beta, msqr = p["mu"], p["bm"], p["beta"], p["msqr"]
    U, S, V = signed_svd(F)
    p0 = bm * (1e-5 + np.sinh(p["xi"] * np.maximum(-log_jp, 0)))
    p_min = -beta * p0
    Je = np.prod(S, -1)
    B = S ** 2
    trB3 = B.sum(-1) / 3
    with np.errstate(invalid="ignore", divide="ignore"):
        Jm = mu * np.power(Je, -2.0 / 3.0)
    sh = Jm[:, None] * (B - trB3[:, None])
    p_trial = -bm * 0.5 * (Je - 1 / Je) * Je
    ysc = 1.5 * (1 + 2 * beta)
    yph = msqr * (p_trial - p_min) * (p_trial - p0)
    s_sq = (sh ** 2).sum(-1)
    y = ysc * s_sq + yph
    hi, lo = p_trial > p0, p_trial < p_min
    proj = ~hi & ~lo & (y >= 1e-4)
    newS = S.copy()
    ljp = log_jp.copy()
    with np.errstate(invalid="ignore", divide="ignore"):
        for mask, pt in ((hi, p0), (lo, p_min)):
            Jn = np.sqrt(-2 * pt / bm + 1)
            newS[mask] = np.cbrt(Jn)[mask, None]
            if p["hardening_on"]:
                ljp[mask] += np.log(Je / Jn)[mask]
        Bs = np.power(Je, 2.0 / 3.0) / mu * np.sqrt(-yph / ysc) / np.sqrt(s_sq)
        newS[proj] = np.sqrt(sh * Bs[:, None] + trB3[:, None])[proj]
        hard = proj & p["hardening_on"] & (p0 > 1e-4) & (p_trial < p0 - 1e-4) & (p_trial > 1e-4 + p_min)
        pc = (1 - beta) * p0 / 2
        q = np.sqrt(1.5 * s_sq)
        d0, d1 = pc - p_trial, -q
        dn = np.hypot(d0, d1)
        d0, d1 = d0 / dn, d1 / dn
        Cq = msqr * (pc - p_min) * (pc - p0)
        Bq = msqr * d0 * (2 * pc - p0 - p_min)
        Aq = msqr * d0 * d0 + (1 + 2 * beta) * d1 * d1
        disc = np.sqrt(Bq * Bq - 4 * Aq * Cq)
        p1, p2 = pc + (-Bq + disc) / (2 * Aq) * d0, pc + (-Bq - disc) / (2 * Aq) * d0
        pf = np.where((p_trial - pc) * (p1 - pc) > 0, p1, p2)
        Jf = np.sqrt(np.abs(-2 * pf / bm + 1))
        upd = hard & (Jf > 1e-4)
        ljp[upd] += np.log(Je / Jf)[upd]
    Fn = np.where((hi | lo | proj)[:, None, None], _udv(U, newS, V), F)
    J = np.prod(newS, -1)
    b = Fn @ np.swapaxes(Fn, -1, -2)
    bd = b - np.trace(b, axis1=1, axis2=2)[:, None, None] / 3 * np.eye(3)
    with np.errstate(invalid="ignore", divide="ignore"):
        dev_c = mu * np.power(J, -2.0 / 3.0)
        i_c = bm * 0.5 * ((J * J - 1) * 0.5 - np.log(J))
    PF = (dev_c[:, None, None] * bd + i_c[:, None, None] * np.eye(3)) * p["volume"]
    rel = lambda a: np.abs(a) / bm  # noqa: E731
    margin = np.minimum.reduce([rel(p_trial - p0), rel(p_trial - p_min), np.abs(y - 1e-4) / (ysc * s_sq + np.abs(yph) + 1e-4)])
    hm = np.minimum.reduce([rel(p0 - 1e-4), rel(p_trial - (p0 - 1e-4)), rel(p_trial - (1e-4 + p_min)), np.abs(Jf - 1e-4)])
    margin = np.where(proj, np.minimum(margin, hm), margin)
    branch = np.select([hi, lo, upd, proj], ["expand", "compress", "project_harden", "project"], "elastic")
    # projections that skip the hardening update only because p0 <= 1e-4 (with beta > 1 the other conditions allow it)
    p0_skip = proj & p["hardening_on"] & (p0 <= 1e-4) & (p_trial < p0 - 1e-4) & (p_trial > 1e-4 + p_min) & (Jf > 1e-4)
    return Fn, PF, ljp, margin, branch, p0_skip


# ---- g2p2g -------------------------------------------------------------------------------------------------------------
def g2p2g(cfg, models, vkeys, vel, vmag, dt, new_dt, near=None):
    """One G2P -> constitutive update -> P2G over all models.

    models: [dict(material, params, state[n,C])]; (vkeys, vel, vmag): grid_update's node velocities and their magnitudes.
    Returns dict(models=[dict(state, pos_mag, f_mag, margin, dropped, lost)], keys, grid[nb,4,64], mag[nb,4,64], stress[nb,4,64]):
    ``mag`` is the per-node magnitude sum M_c of the P2G; ``stress`` sums each particle's stress magnitude (its scale
    (2 mu + lambda) vol |F|^2, for the fluid bulk (gamma + 1) J^-gamma vol J) times its weight and |x_i - x_p| new_dt D^-1,
    the unit in which the tests allow a constitutive model's own error.
    ``near`` [nb, 64] (grid_update's collider info): a particle whose G2P stencil reads a near node is ``tainted``, and so is
    every cell its P2G writes (``taint`` [nb, 64] counts the tainted particles writing a cell)."""
    dx_inv = float(1 << cfg.domain_bits)
    dx = 1.0 / dx_inv
    dinv = 4.0 * dx_inv * dx_inv
    near = np.zeros((len(vkeys), 64), bool) if near is None else np.asarray(near, bool)
    vg = Grid(vkeys, np.concatenate([vel, vmag, near[:, None, :].astype(np.float64)], 1))
    acc = Accumulator(13)
    out = []
    for m in models:
        mat, p = m["material"], m["params"]
        st = np.asarray(m["state"], np.float64)
        n = len(st)
        pos = st[:, :3]
        base, _, W, _, xixp, off = stencil(pos, dx_inv)
        nodes = base[:, None, :] + off[None]
        nv, _ = vg.gather(nodes)
        vi, vim = nv[..., :3], nv[..., 3:6]
        tainted = np.any(nv[..., 6] > 0, axis=1)
        v = np.einsum("nk,nkc->nc", W, vi)
        vm = np.einsum("nk,nkc->nc", W, vim)
        A = np.einsum("nk,nkc,nkd->ncd", W, vi, xixp)
        Am = np.einsum("nk,nkc,nkd->ncd", W, vim, np.abs(xixp))
        xn = pos + v * dt
        pos_mag = np.abs(pos) + vm * dt
        res = dict(margin=np.full(n, np.inf), branch=np.full(n, "elastic"))
        if mat == J_FLUID:
            J0 = st[:, 3]
            J = J0 + np.trace(A, axis1=1, axis2=2) * dt * dinv * J0
            f_mag = np.abs(J0) * (1 + np.trace(Am, axis1=1, axis2=2) * dt * dinv)
            res["margin"] = np.abs(J - 0.1) / 0.1                                   # before the clamp
            J = np.maximum(J, 0.1)
            voln = J * p["volume"]
            pres = p["bulk"] * (np.power(J, -p["gamma"]) - 1)
            PF = (p["viscosity"] * dinv * (A + np.swapaxes(A, 1, 2)) - pres[:, None, None] * np.eye(3)) * voln[:, None, None]
            scale = voln * (p["bulk"] * ((p["gamma"] + 1) * np.power(J, -p["gamma"]) + 1) + 2 * p["viscosity"] * dinv * np.abs(Am).sum((1, 2)))
            new = np.concatenate([xn, J[:, None]], 1)
        else:
            F0 = st[:, 3:12].reshape(n, 3, 3).transpose(0, 2, 1)
            Fg = np.eye(3) + A * dt * dinv
            F = Fg @ F0
            f_mag = (np.eye(3) + Am * dt * dinv) @ np.abs(F0)
            ljp = st[:, 12] if st.shape[1] > 12 else np.zeros(n)
            if mat == FIXED_COROTATED:
                PF = stress_fixed_corotated(p, F)
                Fs, ljs = F, None
            elif mat == SAND:
                Fs, PF, ljs, res["margin"], res["branch"] = stress_sand(p, F, ljp)
            else:
                Fs, PF, ljs, res["margin"], res["branch"], res["p0_skip"] = stress_nacc(p, F, ljp)
            scale = (2 * p["mu"] + p["lambda"] + (p["bm"] if mat == NACC else 0.0)) * p["volume"] * (F ** 2).sum((1, 2))
            cols = [xn, Fs.transpose(0, 2, 1).reshape(n, 9)]
            if ljs is not None:
                cols.append(ljs[:, None])
                f_mag = np.concatenate([f_mag.transpose(0, 2, 1).reshape(n, 9), (np.abs(ljp) + np.abs(ljs) + 1.0)[:, None]], 1)
            else:
                f_mag = f_mag.transpose(0, 2, 1).reshape(n, 9)
            new = np.concatenate(cols, 1)
        D = (A * p["mass"] - PF * new_dt) * dinv
        Dm = (Am * p["mass"] + np.abs(PF) * new_dt) * dinv
        # P2G at the advected position
        nbase, _, W2, G2, xp2, _ = stencil(xn, dx_inv)
        nodes2 = nbase[:, None, :] + off[None]
        ab = ((base - 1) & 3) + 1
        dropped = np.any((ab + nbase - base < 0) | (ab + nbase - base > 5), axis=1)          # quirk #4
        blk = (nbase - 1) >> 2
        G = 1 << (cfg.domain_bits - 2)
        lost = np.any((blk < 0) | (blk >= G) | (np.abs(blk - ((base - 1) >> 2)) > 1), axis=1)   # not re-bucketed
        mass = p["mass"]
        mom = mass * v[:, None, :] + np.einsum("ncd,nkd->nkc", D, xp2)
        # magnitudes: the terms of the sum, and their sensitivity to a relative change 2^-24 of the stored position
        tm = mass * vm[:, None, :] + np.einsum("ncd,nkd->nkc", Dm, np.abs(xp2))
        sens = G2 * (np.abs(xn) * dx_inv).max(1)[:, None]
        tm_s = mass * vm[:, None, :] + np.einsum("ncd,nkd->nkc", Dm, np.abs(xp2) + dx)
        smag = scale[:, None] * new_dt * dinv * np.abs(xp2).sum(-1)
        vals = np.concatenate([
            (mass * W2)[..., None], W2[..., None] * mom,
            (mass * (W2 + sens))[..., None], W2[..., None] * tm + sens[..., None] * tm_s,
            (W2 * smag)[..., None].repeat(4, -1) * np.array([0, 1, 1, 1.0]),
            np.broadcast_to(tainted[:, None, None], W2.shape + (1,)).astype(np.float64)], -1)
        acc.add(nodes2, vals, in_domain_nodes(cfg, nodes2) & ~dropped[:, None])
        res.update(state=new, pos_mag=pos_mag, f_mag=f_mag, dropped=dropped, lost=lost, stress_scale=scale,
                   v=v, v_mag=vm, cell=nbase - 1, tainted=tainted)
        out.append(res)
    keys, g = acc.result()
    return dict(models=out, keys=keys, grid=g[:, :4], mag=g[:, 4:8], stress=g[:, 8:12], taint=g[:, 12])


def substep(cfg, models, keys, grid, dt, dt_default, time_left=np.inf, collider=None, t=0.0, objects=None):
    """The whole sub-step: grid update at dt (with ``collider`` = (col, sdf, grad), then ``objects``, placed at the float32
    time t), new_dt from its max, g2p2g with (dt, new_dt).  ``dt_range`` = (new_dt of mx_hi, new_dt of mx_lo): the new dt over
    every branch choice of the near nodes; ``collider_info`` is grid_update's."""
    u = grid_update(cfg, keys, grid, dt, collider, t, objects)
    vel, vmag, mx = u[:3]
    info = u[3] if len(u) > 3 else dict(near=None, mx_lo=mx, mx_hi=mx, mx_err=0.0)
    new_dt = compute_dt(cfg, mx, dt_default, time_left)
    r = g2p2g(cfg, models, keys, vel, vmag, dt, new_dt, info["near"])
    r.update(max_vsq=mx, new_dt=new_dt, vel=vel, vel_mag=vmag, collider_info=info,
             dt_range=(compute_dt(cfg, info["mx_hi"], dt_default, time_left), compute_dt(cfg, info["mx_lo"], dt_default, time_left)))
    return r


# ---- comparison ----------------------------------------------------------------------------------------------------------
def cell_overflow(res, max_ppc):
    """g2p2g's cell capacity: each model's particles re-bucket into their new cell (``res["cell"]``, lost ones excepted),
    and a cell takes at most ``max_ppc`` of them.  The others are left out of the next partition; which ones depends on
    the order of the atomics.  Their P2G of this sub-step still happens.
    Returns (over[n]: the particle's new cell holds more than max_ppc, number of such cells, particles kept)."""
    keep = ~res["lost"]
    cells = key_hash(res["cell"][keep] + 1)          # + 1: a cell of a kept particle is >= -1
    _, inv, cnt = np.unique(cells, return_inverse=True, return_counts=True)
    over = np.zeros(len(keep), bool)
    over[np.flatnonzero(keep)] = cnt[inv] > max_ppc
    return over, int((cnt > max_ppc).sum()), int(np.minimum(cnt, max_ppc).sum())


def compare(ref, keys, grid, states, kappa, stress_allow, f_allow, margin=1e-4, match_tol=1e-5, max_ppc=None):
    """Worst ratio |impl - ref64| / bound of every quantity (<= 1 passes) for one sub-step's outputs of an implementation:
    ``keys``/``grid`` its keyed grid after the sub-step, ``states`` its particle_state rows per model.
    bound = kappa[q] * 2^-24 * M (+ stress_allow[model] * the stress column of the node, + f_allow[model] for F / logJp).
    Particles within ``margin`` of a return-mapping branch are left out of the particle check and counted.  With
    ``max_ppc``, a new cell that ref64 gives more than max_ppc particles must hold exactly max_ppc of them (cell_overflow);
    the grid includes every particle's P2G either way."""
    rep = dict(mass=0.0, momentum=0.0, pos=0.0, F=0.0, near_branch=0, worst={}, tainted_cells=0, tainted_particles=0)
    keys = np.asarray(keys, np.int64)
    grid = np.asarray(grid, np.float64)
    # every block of the reference's P2G must exist; blocks the reference never touched must be zero
    eh = key_hash(keys)
    rh = key_hash(ref["keys"])
    touched = ref["grid"][:, 0].max(1) > 0
    missing = np.setdiff1d(rh[touched], eh)
    assert len(missing) == 0, f"{len(missing)} grid blocks with mass missing from the implementation's grid"
    val, mag, st = ref_at(ref, keys)
    err = np.abs(grid - val)
    if "taint" in ref:   # cells written by a particle that read a collider node near a discontinuity
        taint, _ = Grid(ref["keys"], ref["taint"][:, None, :]).gather(np.asarray(keys, np.int64)[:, None, :] * 4 + _CELLS[None])
        bad = taint[..., 0] > 0
        rep["tainted_cells"] = int(bad.sum())
        err = np.where(bad[:, None, :], 0.0, err)
    bm = kappa["mass"] * EPS32 * mag[:, 0]
    bmv = kappa["momentum"] * EPS32 * mag[:, 1:] + stress_allow * st[:, 1:]
    with np.errstate(divide="ignore", invalid="ignore"):
        rm = np.where(err[:, 0] > 0, err[:, 0] / bm, 0.0)
        rmv = np.where(err[:, 1:] > 0, err[:, 1:] / bmv, 0.0)
    rep["mass"], rep["momentum"] = float(np.nan_to_num(rm, nan=np.inf).max(initial=0)), float(np.nan_to_num(rmv, nan=np.inf).max(initial=0))
    if rep["momentum"] > 1 or rep["mass"] > 1:
        i = np.unravel_index(np.argmax(np.nan_to_num(rmv, nan=np.inf)), rmv.shape)
        rep["worst"]["momentum"] = (tuple(int(k) for k in keys[i[0]]), int(i[2]), float(grid[i[0], 1 + i[1], i[2]]), float(val[i[0], 1 + i[1], i[2]]), float(bmv[i]))
    compare_particles(ref["models"], states, kappa, f_allow, margin, match_tol, rep, max_ppc)
    return rep


def ref_at(ref, keys):
    """The reference's (value, magnitude, stress column) [nb, 4, 64] at the blocks ``keys`` (0 where it touched nothing)."""
    rg = Grid(ref["keys"], np.concatenate([ref["grid"], ref["mag"], ref["stress"]], 1))
    cells = np.stack(np.meshgrid(np.arange(4), np.arange(4), np.arange(4), indexing="ij"), -1).reshape(64, 3)
    nodes = np.asarray(keys, np.int64)[:, None, :] * 4 + cells[None]
    r, _ = rg.gather(nodes)                                  # [nb, 64, 12]
    r = r.transpose(0, 2, 1)
    return r[:, :4], r[:, 4:8], r[:, 8:12]


def compare_particles(ref_models, states, kappa, f_allow, margin, match_tol, rep, max_ppc=None):
    """compare()'s per-particle rules: ``states[m]`` against ``ref_models[m]`` (lost particles left out), worst ratios into rep.
    Every implementation particle is matched by position to its own reference particle.  The count must be the
    reference's: n - lost, and with ``max_ppc`` each overflowing cell (cell_overflow) holding exactly max_ppc particles."""
    from scipy.spatial import cKDTree
    for m, (res, se) in enumerate(zip(ref_models, states)):
        keep = ~res["lost"]
        if max_ppc is None:
            over, n_over, want = np.zeros(len(keep), bool), 0, int(keep.sum())
        else:
            over, n_over, want = cell_overflow(res, max_ppc)
        rs = res["state"][keep]
        assert len(se) == want, (f"model {m}: {len(se)} particles, reference keeps {want} ({int((~keep).sum())} lost, "
                                 f"{n_over} cells over max_ppc = {max_ppc})")
        if len(rs) == 0:
            continue
        se = np.asarray(se, np.float64)
        d, idx = cKDTree(rs[:, :3]).query(se[:, :3], k=1)
        assert d.max() <= match_tol and len(np.unique(idx)) == len(se), f"model {m}: particles do not match by position ({d.max():.3e})"
        ov = over[keep]
        assert np.all(np.isin(np.flatnonzero(~ov), idx)), f"model {m}: a particle outside the overflowing cells is missing"
        if n_over:
            held = key_hash(res["cell"][keep][idx[ov[idx]]] + 1)
            _, cnt = np.unique(held, return_counts=True)
            assert len(cnt) == n_over and np.all(cnt == max_ppc), f"model {m}: overflowing cells hold {sorted(cnt.tolist())}, want {n_over} x {max_ppc}"
        rs = rs[idx]
        tainted = res["tainted"][keep][idx] if "tainted" in res else np.zeros(len(idx), bool)
        rep["tainted_particles"] = rep.get("tainted_particles", 0) + int(tainted.sum())
        rp = np.where(tainted[:, None], 0.0, np.abs(se[:, :3] - rs[:, :3]) / (kappa["pos"] * EPS32 * res["pos_mag"][keep][idx]))
        rep["pos"] = max(rep["pos"], float(rp.max()))
        if rs.shape[1] > 3:
            near = res["margin"][keep][idx] < margin
            rep["near_branch"] += int(near.sum())
            fm = res["f_mag"][keep][idx] if res["f_mag"].ndim > 1 else res["f_mag"][keep][idx][:, None]
            ef = np.abs(se[:, 3:] - rs[:, 3:])
            with np.errstate(divide="ignore", invalid="ignore"):
                rf = np.where(ef > 0, ef / (kappa["F"] * EPS32 * fm + f_allow[m]), 0.0)
            rep["F"] = max(rep["F"], float(rf[~near & ~tainted].max(initial=0)))
