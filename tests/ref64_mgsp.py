"""The float64 reference (tests/ref64.py) for MGSP ranks: one sub-step of every rank's shard, compared per grid copy and per
particle.

A rank holds the particle and neighbour blocks of its own particles.  A block shared by several ranks must hold the full sum
on every owner (DESIGN.md section 6), with one exception: a block that enters a rank's partition in a sub-step is tagged as
shared only at the end of that sub-step, so that rank's copy holds zeros for one sub-step ("fresh").  That is correct only if
no particle of the rank reads it at its next G2P; compare() asserts exactly that, from the stencils.

Input per rank: dict(keys[nb, 3], grid[nb, 4, 64], models=[dict(model=<scene model index>, material, params, state)]), the
rank's view before the sub-step.  The reference feeds every rank's particles from that rank's own grid copies, with fresh
copies replaced by the full sum another owner holds: a rank that reads a fresh copy then misses its particle bounds.
"""
import numpy as np

import ref64
from ref64 import EPS32, key_hash

# A halo cell is the sum of one FP32 partial sum per owner, so each remote add is one more rounding.  The FP32 oracle's cells
# with 2 to 4 owners stay within the single-domain kappa all the same (test_ref64_mgsp_cpu.py asserts it and prints the worst
# ratio), so every copy is held to that kappa with no halo allowance.

_CELLS = np.stack(np.meshgrid(np.arange(4), np.arange(4), np.arange(4), indexing="ij"), -1).reshape(64, 3)
_OFF = np.stack(np.meshgrid(np.arange(3), np.arange(3), np.arange(3), indexing="ij"), -1).reshape(27, 3)


def _dx_inv(cfg):
    return float(1 << cfg.domain_bits)


def stencil_blocks(cfg, pos):
    """Key hashes [n, 27] of the grid blocks a particle at pos reads at its G2P (-1 for a node outside the domain)."""
    base = ref64.cell_index(np.asarray(pos, np.float64).reshape(-1, 3), _dx_inv(cfg)) - 1
    nodes = base[:, None, :] + _OFF[None]
    return np.where(ref64.in_domain_nodes(cfg, nodes), key_hash(nodes >> 2), -1)


def partition_keys(cfg, pos):
    """The keys [k, 3] of the particle blocks of ``pos`` and their 2x2x2 neighbourhoods (a rank's partition)."""
    base = ref64.cell_index(np.asarray(pos, np.float64).reshape(-1, 3), _dx_inv(cfg)) - 1
    blk = (base - 1) >> 2
    G = 1 << (cfg.domain_bits - 2)
    nb = (blk[:, None, :] + _OFF[None, np.all(_OFF < 2, axis=1)]).reshape(-1, 3)
    nb = nb[np.all((nb >= 0) & (nb < G), axis=1)]
    return np.unique(nb, axis=0)


def _sum_keyed(parts, nch):
    """Key-wise sum of [(keys, data[nb, nch, 64])] -> (keys, sum, number of parts with data[:, 0] > 0 per cell [nb, 64])."""
    parts = [(np.asarray(k, np.int64).reshape(-1, 3), np.asarray(d, np.float64)) for k, d in parts]
    if not parts or sum(len(k) for k, _ in parts) == 0:
        return np.zeros((0, 3), np.int64), np.zeros((0, nch, 64)), np.zeros((0, 64), np.int64)
    keys = np.concatenate([k for k, _ in parts])
    data = np.concatenate([d for _, d in parts])
    h = key_hash(keys)
    uh, first, inv = np.unique(h, return_index=True, return_inverse=True)
    out = np.zeros((len(uh), nch, 64))
    np.add.at(out, inv, data)
    owners = np.zeros((len(uh), 64), np.int64)
    np.add.at(owners, inv, (data[:, 0] > 0).astype(np.int64))
    return keys[first], out, owners


def _fill_fresh(ranks):
    """Every rank's grid with its all-zero copies replaced by a non-zero copy of the same key from another rank."""
    hs = [key_hash(np.asarray(r["keys"], np.int64).reshape(-1, 3)) for r in ranks]
    full = {}
    for ri, (r, h) in enumerate(zip(ranks, hs)):
        nz = np.abs(np.asarray(r["grid"])).reshape(len(h), -1).max(1, initial=0) > 0
        for b in np.nonzero(nz)[0]:
            full.setdefault(int(h[b]), (ri, int(b)))
    views, n = [], 0
    for ri, (r, h) in enumerate(zip(ranks, hs)):
        v = np.array(r["grid"], np.float64).reshape(len(h), 4, 64)
        zero = np.abs(v).reshape(len(h), -1).max(1, initial=0) == 0
        for b in np.nonzero(zero)[0]:
            src = full.get(int(h[b]))
            if src is not None and src[0] != ri:
                v[b] = ranks[src[0]]["grid"][src[1]]
                n += 1
        views.append(v)
    return views, n


def _union_models(per_rank, n_models):
    """Per scene model, the concatenation of every rank's part (ref64.g2p2g's per-model results, in rank order)."""
    out = []
    for gm in range(n_models):
        got = [res for r in per_rank for m, res in r if m == gm]
        if not got:
            out.append(None)
            continue
        u = {}
        for f in ("state", "pos_mag", "f_mag", "margin", "branch", "dropped", "lost", "tainted"):
            u[f] = np.concatenate([g[f] for g in got])
        out.append(u)
    return out


def substep(cfg, ranks, dt, dt_default, time_left=np.inf, n_models=None, collider=None, t=0.0, objects=None):
    """The reference sub-step of all ranks: every rank's grid update and g2p2g on its own view (fresh copies filled), the
    next grid summed key-wise over the ranks (magnitudes and stress columns likewise), new_dt from the max over the ranks'
    maxima.  ``collider`` = (col, sdf, grad) and then ``objects`` act in every rank's grid update at the float32 time t
    (ref64.grid_update); the
    engine's ranks agree on a max their next-max predictor computed at the end of the previous sub-step, at the time this
    grid update sees.  Returns a dict ref64.compare-like (keys, grid, mag, stress, models per scene model, new_dt) plus owners
    (contributing ranks per cell), pre_keys (every rank's key hashes before the sub-step), fresh_in (copies filled), and per
    rank its models' results (per_rank: [(scene model, result)]) and its P2G (partials: (keys, grid))."""
    views, fresh_in = _fill_fresh(ranks)
    ups = [ref64.grid_update(cfg, r["keys"], v, dt, collider, t, objects) for r, v in zip(ranks, views)]
    mx = max((u[2] for u in ups), default=0.0)
    new_dt = ref64.compute_dt(cfg, mx, dt_default, time_left)
    infos = [u[3] if len(u) > 3 else dict(near=None, mx_lo=u[2], mx_hi=u[2], mx_err=0.0) for u in ups]
    mx_lo, mx_hi = max((i["mx_lo"] for i in infos), default=0.0), max((i["mx_hi"] for i in infos), default=0.0)
    mx_err = max((i["mx_err"] for i in infos), default=0.0)
    if n_models is None:
        n_models = 1 + max((m["model"] for r in ranks for m in r["models"]), default=-1)
    parts, per_rank = [], []
    for r, u, info in zip(ranks, ups, infos):
        res = ref64.g2p2g(cfg, r["models"], r["keys"], u[0], u[1], dt, new_dt, info["near"])
        parts.append((res["keys"], np.concatenate([res["grid"], res["mag"], res["stress"], res["taint"][:, None]], 1)))
        per_rank.append([(m["model"], mr) for m, mr in zip(r["models"], res["models"])])
    keys, s, owners = _sum_keyed(parts, 13)
    return dict(keys=keys, grid=s[:, :4], mag=s[:, 4:8], stress=s[:, 8:12], taint=s[:, 12], owners=owners, models=_union_models(per_rank, n_models),
                new_dt=new_dt, max_vsq=mx, near=sum(int(i["near"].sum()) for i in infos if i["near"] is not None),
                mx_hi=mx_hi, mx_lo=mx_lo, mx_err=mx_err, dt_range=(ref64.compute_dt(cfg, mx_hi, dt_default, time_left), ref64.compute_dt(cfg, mx_lo, dt_default, time_left)), fresh_in=fresh_in, per_rank=per_rank, partials=[(k, d[:, :4]) for k, d in parts], pre_keys=[set(key_hash(np.asarray(r["keys"], np.int64).reshape(-1, 3)).tolist()) for r in ranks])


def rasterize(cfg, ranks_models):
    """The set-up grid: ref64.rasterize of every rank's particles, summed key-wise (ranks_models: per rank [dict(pos, v0, mass)])."""
    parts = []
    for ms in ranks_models:
        k, g, m = ref64.rasterize(cfg, ms)
        parts.append((k, np.concatenate([g, m], 1)))
    keys, s, owners = _sum_keyed(parts, 8)
    return dict(keys=keys, grid=s[:, :4], mag=s[:, 4:8], stress=np.zeros_like(s[:, :4]), owners=owners, models=[], pre_keys=None)


def _ref_at(ref, keys):
    rg = ref64.Grid(ref["keys"], np.concatenate([ref["grid"], ref["mag"], ref["stress"], ref["owners"][:, None, :]], 1))
    r, _ = rg.gather(np.asarray(keys, np.int64)[:, None, :] * 4 + _CELLS[None])
    r = r.transpose(0, 2, 1)
    return r[:, :4], r[:, 4:8], r[:, 8:12], r[:, 12]


def _readers(cfg, states):
    """key hash -> (scene model, row, position) of the first particle whose next G2P stencil reads that block."""
    out = {}
    for gm, s in sorted(states.items()):
        s = np.asarray(s)
        if len(s) == 0:
            continue
        h = stencil_blocks(cfg, s[:, :3])
        u, i = np.unique(h.reshape(-1), return_index=True)
        for hh, ii in zip(u.tolist(), (i // 27).tolist()):
            if hh >= 0:
                out.setdefault(hh, (gm, ii, tuple(float(x) for x in s[ii, :3])))
    return out


def _key(h):
    return (h >> 40, (h >> 20) & 0xFFFFF, h & 0xFFFFF)


def compare(cfg, ref, after, kappa, stress_allow, f_allow, margin=1e-4, match_tol=1e-5):
    """Worst ratio |rank copy - ref| / bound per quantity (<= 1 passes) for every copy on every rank, then the union of the ranks'
    particles per scene model with ref64's per-particle rules.  ``after``: per rank dict(keys, grid, states={model: rows}).
    bound = kappa * 2^-24 * M (+ stress_allow * the stress column), the single-domain bound, also on cells with several owners.
    Every block a rank's particle reads at its next G2P must be among that rank's keys.  A rank's copy may be all zero only if the key was not in that rank's partition before the sub-step, another rank holds a
    non-zero copy and no particle of that rank reads the block at its next G2P; anything else raises AssertionError naming the
    block.  Also: every block the reference touches has a non-fresh copy somewhere.
    Returns dict(mass, momentum, pos, F, near_branch, worst, fresh, max_owners, shared)."""
    rep = dict(mass=0.0, momentum=0.0, pos=0.0, F=0.0, near_branch=0, worst={}, fresh=0, max_owners=0, shared=0, tainted_cells=0)
    hs = [key_hash(np.asarray(a["keys"], np.int64).reshape(-1, 3)) for a in after]
    nonzero = [np.abs(np.asarray(a["grid"], np.float64)).reshape(len(h), -1).max(1, initial=0) > 0 for a, h in zip(after, hs)]
    holders = {}
    for ri, (h, nz) in enumerate(zip(hs, nonzero)):
        for hh, z in zip(h.tolist(), nz.tolist()):
            holders.setdefault(hh, []).append((ri, z))
    rep["max_owners"] = max((len(v) for v in holders.values()), default=0)
    rep["shared"] = sum(len(v) > 1 for v in holders.values())
    ref_touched = set(key_hash(ref["keys"][np.abs(ref["grid"]).reshape(len(ref["keys"]), -1).max(1, initial=0) > 0]).tolist())
    good = set()
    for ri, (a, h, nz) in enumerate(zip(after, hs, nonzero)):
        keys = np.asarray(a["keys"], np.int64).reshape(-1, 3)
        grid = np.asarray(a["grid"], np.float64).reshape(len(keys), 4, 64)
        val, mag, st, own = _ref_at(ref, keys)
        fresh = np.zeros(len(keys), bool)
        readers = _readers(cfg, a.get("states", {}))
        have = set(h.tolist())
        for hh, rd in readers.items():
            assert hh in have, f"rank {ri} block {_key(hh)}: missing from the rank's keys, but particle {rd[1]} of model {rd[0]} at {rd[2]} reads it at its next G2P"
        for b in np.nonzero(~nz)[0]:
            hh = int(h[b])
            if hh not in ref_touched:
                continue
            where = f"rank {ri} block {_key(hh)}"
            pre = ref["pre_keys"]
            assert pre is not None and hh not in pre[ri], f"{where}: all zero, but it was in the rank's partition before the sub-step (the reference holds mass {val[b, 0].sum():.3e})"
            assert any(z for r2, z in holders[hh] if r2 != ri), f"{where}: all zero and no other rank holds a non-zero copy"
            rd = readers.get(hh)
            assert rd is None, f"{where}: all zero (fresh), but particle {rd[1]} of model {rd[0]} at {rd[2]} reads it at its next G2P"
            fresh[b] = True
        rep["fresh"] += int(fresh.sum())
        good |= set(h[~fresh].tolist())
        err = np.abs(grid - val)
        if "taint" in ref:   # cells written by a particle that read a collider node near a discontinuity (ref64.g2p2g)
            taint, _ = ref64.Grid(ref["keys"], ref["taint"][:, None, :]).gather(keys[:, None, :] * 4 + _CELLS[None])
            bad = (taint[..., 0] > 0) & ~fresh[:, None]
            rep["tainted_cells"] += int(bad.sum())
            err = np.where(bad[:, None, :], 0.0, err)
        err = err[~fresh]
        bm = kappa["mass"] * EPS32 * mag[~fresh, 0]
        bmv = kappa["momentum"] * EPS32 * mag[~fresh, 1:] + stress_allow * st[~fresh, 1:]
        with np.errstate(divide="ignore", invalid="ignore"):
            rm = np.nan_to_num(np.where(err[:, 0] > 0, err[:, 0] / bm, 0.0), nan=np.inf)
            rmv = np.nan_to_num(np.where(err[:, 1:] > 0, err[:, 1:] / bmv, 0.0), nan=np.inf)
        for q, ratio, ch in (("mass", rm, lambda i: (0, i[1])), ("momentum", rmv, lambda i: (1 + i[1], i[2]))):
            w = float(ratio.max(initial=0))
            if w > rep[q]:
                rep[q] = w
                if w > 1:
                    i = np.unravel_index(np.argmax(ratio), ratio.shape)
                    b = np.nonzero(~fresh)[0][i[0]]
                    c, cell = ch(i)
                    rep["worst"][q] = dict(rank=ri, block=tuple(int(k) for k in keys[b]), channel=c, cell=int(cell), owners=int(own[b, cell]),
                                           value=float(grid[b, c, cell]), ref=float(val[b, c, cell]), ratio=w)
    lacking = ref_touched - good
    assert not lacking, f"{len(lacking)} blocks the reference touches have no non-fresh copy on any rank, e.g. {_key(next(iter(lacking)))}"
    if ref["models"]:
        states = []
        for gm in range(len(ref["models"])):
            rows = [np.asarray(a["states"][gm]) for a in after if gm in a.get("states", {})]
            states.append(np.concatenate(rows) if rows else np.zeros((0, 3), np.float32))
        models = [m if m is not None else dict(state=np.zeros((0, 3)), lost=np.zeros(0, bool)) for m in ref["models"]]
        ref64.compare_particles(models, states, kappa, f_allow, margin, match_tol, rep)
    return rep


def check_dts(dts, ref_dt, ulps):
    """Every rank's dt bit-identical, and within ``ulps`` float32 ulps of the reference's new_dt."""
    d = np.asarray(dts, np.float32)
    assert np.all(d.view(np.int32) == d[0].view(np.int32)), f"the ranks' dt differ: {[float(x) for x in d]}"
    ulp = float(np.spacing(np.float32(ref_dt)))
    assert abs(float(d[0]) - ref_dt) <= ulps * ulp, f"dt {float(d[0])!r} vs reference {ref_dt!r} ({(float(d[0]) - ref_dt) / ulp:.2f} ulp)"
