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
* nodes outside the domain do not exist: what a particle would add there is dropped.

Every output comes with a magnitude M such that an FP32 implementation of the same operations differs from the float64
value by at most a small multiple of 2^-24 * M.  The tests fix that multiple (kappa) per quantity.
"""
import numpy as np

J_FLUID, FIXED_COROTATED, SAND, NACC = 0, 1, 2, 3
CHANNELS = {J_FLUID: 4, FIXED_COROTATED: 12, SAND: 13, NACC: 13}
EPS32 = 2.0 ** -24


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


def grid_update(cfg, keys, grid, dt):
    """v = mv / m, wall mask on both faces (key < boundary or key >= G - boundary), then gravity.
    Returns (vel[nb,3,64] (0 where m = 0), magnitude[nb,3,64], max |v|^2 with NaN -> +inf)."""
    keys = np.asarray(keys, np.int64)
    grid = np.asarray(grid, np.float64)
    G, bc = 1 << (cfg.domain_bits - 2), cfg.boundary
    wall = (keys < bc) | (keys >= G - bc)                       # [nb, 3]
    m = grid[:, 0]
    has = m > 0
    with np.errstate(divide="ignore", invalid="ignore"):
        v = np.where(has[:, None], grid[:, 1:] / np.where(has, m, 1.0)[:, None], 0.0)
    v = np.where(wall[:, :, None], 0.0, v)
    mag = np.abs(v).copy()
    gdt = float(np.float32(cfg.gravity)) * dt
    v[:, 1] += np.where(has, gdt, 0.0)
    mag[:, 1] += np.where(has, abs(gdt), 0.0)
    vsq = (v ** 2).sum(1)
    vsq = np.where(np.isnan(vsq), np.inf, vsq)
    return v, mag, float(vsq.max()) if vsq.size else 0.0


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
    return Fn, PF, ljp, margin, branch


# ---- g2p2g -------------------------------------------------------------------------------------------------------------
def g2p2g(cfg, models, vkeys, vel, vmag, dt, new_dt):
    """One G2P -> constitutive update -> P2G over all models.

    models: [dict(material, params, state[n,C])]; (vkeys, vel, vmag): grid_update's node velocities and their magnitudes.
    Returns dict(models=[dict(state, pos_mag, f_mag, margin, dropped, lost)], keys, grid[nb,4,64], mag[nb,4,64], stress[nb,4,64]):
    ``mag`` is the per-node magnitude sum M_c of the P2G; ``stress`` sums each particle's stress magnitude (its scale
    (2 mu + lambda) vol |F|^2, for the fluid bulk (gamma + 1) J^-gamma vol J) times its weight and |x_i - x_p| new_dt D^-1,
    the unit in which the tests allow a constitutive model's own error."""
    dx_inv = float(1 << cfg.domain_bits)
    dx = 1.0 / dx_inv
    dinv = 4.0 * dx_inv * dx_inv
    vg = Grid(vkeys, np.concatenate([vel, vmag], 1))
    acc = Accumulator(12)
    out = []
    for m in models:
        mat, p = m["material"], m["params"]
        st = np.asarray(m["state"], np.float64)
        n = len(st)
        pos = st[:, :3]
        base, _, W, _, xixp, off = stencil(pos, dx_inv)
        nodes = base[:, None, :] + off[None]
        nv, _ = vg.gather(nodes)
        vi, vim = nv[..., :3], nv[..., 3:]
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
                Fs, PF, ljs, res["margin"], res["branch"] = stress_nacc(p, F, ljp)
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
            (W2 * smag)[..., None].repeat(4, -1) * np.array([0, 1, 1, 1.0])], -1)
        acc.add(nodes2, vals, in_domain_nodes(cfg, nodes2) & ~dropped[:, None])
        res.update(state=new, pos_mag=pos_mag, f_mag=f_mag, dropped=dropped, lost=lost, stress_scale=scale,
                   v=v, v_mag=vm)
        out.append(res)
    keys, g = acc.result()
    return dict(models=out, keys=keys, grid=g[:, :4], mag=g[:, 4:8], stress=g[:, 8:12])


def substep(cfg, models, keys, grid, dt, dt_default, time_left=np.inf):
    """The whole sub-step: grid update at dt, new_dt from its max, g2p2g with (dt, new_dt)."""
    vel, vmag, mx = grid_update(cfg, keys, grid, dt)
    new_dt = compute_dt(cfg, mx, dt_default, time_left)
    r = g2p2g(cfg, models, keys, vel, vmag, dt, new_dt)
    r.update(max_vsq=mx, new_dt=new_dt, vel=vel, vel_mag=vmag)
    return r


# ---- comparison ----------------------------------------------------------------------------------------------------------
def compare(ref, keys, grid, states, kappa, stress_allow, f_allow, margin=1e-4, match_tol=1e-5):
    """Worst ratio |impl - ref64| / bound of every quantity (<= 1 passes) for one sub-step's outputs of an implementation:
    ``keys``/``grid`` its keyed grid after the sub-step, ``states`` its particle_state rows per model.
    bound = kappa[q] * 2^-24 * M (+ stress_allow[model] * the stress column of the node, + f_allow[model] for F / logJp).
    Particles within ``margin`` of a return-mapping branch are left out of the particle check and counted."""
    rep = dict(mass=0.0, momentum=0.0, pos=0.0, F=0.0, near_branch=0, worst={})
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
    bm = kappa["mass"] * EPS32 * mag[:, 0]
    bmv = kappa["momentum"] * EPS32 * mag[:, 1:] + stress_allow * st[:, 1:]
    with np.errstate(divide="ignore", invalid="ignore"):
        rm = np.where(err[:, 0] > 0, err[:, 0] / bm, 0.0)
        rmv = np.where(err[:, 1:] > 0, err[:, 1:] / bmv, 0.0)
    rep["mass"], rep["momentum"] = float(np.nan_to_num(rm, nan=np.inf).max(initial=0)), float(np.nan_to_num(rmv, nan=np.inf).max(initial=0))
    if rep["momentum"] > 1 or rep["mass"] > 1:
        i = np.unravel_index(np.argmax(np.nan_to_num(rmv, nan=np.inf)), rmv.shape)
        rep["worst"]["momentum"] = (tuple(int(k) for k in keys[i[0]]), int(i[2]), float(grid[i[0], 1 + i[1], i[2]]), float(val[i[0], 1 + i[1], i[2]]), float(bmv[i]))
    compare_particles(ref["models"], states, kappa, f_allow, margin, match_tol, rep)
    return rep


def ref_at(ref, keys):
    """The reference's (value, magnitude, stress column) [nb, 4, 64] at the blocks ``keys`` (0 where it touched nothing)."""
    rg = Grid(ref["keys"], np.concatenate([ref["grid"], ref["mag"], ref["stress"]], 1))
    cells = np.stack(np.meshgrid(np.arange(4), np.arange(4), np.arange(4), indexing="ij"), -1).reshape(64, 3)
    nodes = np.asarray(keys, np.int64)[:, None, :] * 4 + cells[None]
    r, _ = rg.gather(nodes)                                  # [nb, 64, 12]
    r = r.transpose(0, 2, 1)
    return r[:, :4], r[:, 4:8], r[:, 8:12]


def compare_particles(ref_models, states, kappa, f_allow, margin, match_tol, rep):
    """compare()'s per-particle rules: ``states[m]`` against ``ref_models[m]`` (lost particles left out), worst ratios into rep."""
    from scipy.spatial import cKDTree
    for m, (res, se) in enumerate(zip(ref_models, states)):
        keep = ~res["lost"]
        rs = res["state"][keep]
        assert len(se) == len(rs), f"model {m}: {len(se)} particles, reference keeps {len(rs)}"
        if len(rs) == 0:
            continue
        d, idx = cKDTree(np.asarray(se, np.float64)[:, :3]).query(rs[:, :3], k=1)
        assert d.max() <= match_tol and len(np.unique(idx)) == len(rs), f"model {m}: particles do not match by position ({d.max():.3e})"
        e = np.asarray(se, np.float64)[idx]
        rp = np.abs(e[:, :3] - rs[:, :3]) / (kappa["pos"] * EPS32 * res["pos_mag"][keep])
        rep["pos"] = max(rep["pos"], float(rp.max()))
        if rs.shape[1] > 3:
            near = res["margin"][keep] < margin
            rep["near_branch"] += int(near.sum())
            fm = res["f_mag"][keep] if res["f_mag"].ndim > 1 else res["f_mag"][keep][:, None]
            ef = np.abs(e[:, 3:] - rs[:, 3:])
            with np.errstate(divide="ignore", invalid="ignore"):
                rf = np.where(ef > 0, ef / (kappa["F"] * EPS32 * fm + f_allow[m]), 0.0)
            rep["F"] = max(rep["F"], float(rf[~near].max(initial=0)))
