"""float64 numpy restatement of the level-set samplers (include/claymore_b200.h, DESIGN §2.7), independent of the library.

    philox4x32_10(ctr, key)            Philox4x32-10 on (N, 4) uint32 counters
    valid_cells(n, phi)                ascending ids i + (ni-1)(j + (nj-1) k) of the cells with a negative node
    trilinear(n, phi, x, y, z)         fetchGridTrilinear (SampleGenerator.h:30-53) in float64
    sample_random / sample_lattice     the rows of cb200_sample_sdf, in order
    text(n, h, phi)                    SDFGen text of a float32 field (9 significant digits: strtof gives back the same floats)
plus a few synthetic level sets for the tests.
"""
import numpy as np

_MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: (N, 4) uint32, key: (2,) uint32 -> (N, 4) uint32 (Salmon et al., SC 2011)."""
    c = [np.asarray(ctr, np.uint64)[:, i].copy() for i in range(4)]
    k0, k1 = np.uint64(int(key[0]) & 0xFFFFFFFF), np.uint64(int(key[1]) & 0xFFFFFFFF)
    for r in range(10):
        if r:
            k0 = (k0 + np.uint64(0x9E3779B9)) & _MASK
            k1 = (k1 + np.uint64(0xBB67AE85)) & _MASK
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _MASK, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _MASK]
    return np.stack(c, 1).astype(np.uint32)


def text(n, h, phi, origin=(0.0, 0.0, 0.0)):
    """SDFGen text: phi is indexed [k, j, i] (or flat with i fastest)."""
    vals = np.asarray(phi, np.float32).reshape(-1)
    head = f"{n[0]} {n[1]} {n[2]}\n{origin[0]!r} {origin[1]!r} {origin[2]!r}\n{float(np.float32(h))!r}\n"
    return (head + "\n".join(f"{v:.9g}" for v in vals) + "\n").encode()


def node_box(n, h, offset, span):
    h = float(np.float32(h))
    s = min(float(span[d]) / (float(n[d] - 1) * h) for d in range(3))
    c = s * h
    return c, [float(offset[d]) for d in range(3)], [float(offset[d]) + float(n[d] - 1) * c for d in range(3)]


def valid_cells(n, phi):
    g = np.asarray(phi, np.float32).reshape(n[2], n[1], n[0]) < 0
    m = np.zeros((n[2] - 1, n[1] - 1, n[0] - 1), bool)
    for a in (0, 1):
        for b in (0, 1):
            for c in (0, 1):
                m |= g[a:a + n[2] - 1, b:b + n[1] - 1, c:c + n[0] - 1]
    return np.flatnonzero(m.reshape(-1))


def trilinear(n, phi, x, y, z):
    p = np.asarray(phi, np.float32).reshape(-1).astype(np.float64)
    at = lambda i, j, k: p[i + n[0] * (j + n[1] * k)]
    fx, fy, fz = np.floor(x), np.floor(y), np.floor(z)
    dx, dy, dz = x - fx, y - fy, z - fz
    x0, y0, z0 = fx.astype(np.int64), fy.astype(np.int64), fz.astype(np.int64)
    x1, y1, z1 = np.ceil(x).astype(np.int64), np.ceil(y).astype(np.int64), np.ceil(z).astype(np.int64)
    c000, c001, c010, c011 = at(x0, y0, z0), at(x0, y0, z1), at(x0, y1, z0), at(x0, y1, z1)
    c100, c101, c110, c111 = at(x1, y0, z0), at(x1, y0, z1), at(x1, y1, z0), at(x1, y1, z1)
    c00 = c000 * (1 - dx) + c100 * dx
    c01 = c001 * (1 - dx) + c101 * dx
    c10 = c010 * (1 - dx) + c110 * dx
    c11 = c011 * (1 - dx) + c111 * dx
    c0 = c00 * (1 - dy) + c10 * dy
    c1 = c01 * (1 - dy) + c11 * dy
    return c0 * (1 - dz) + c1 * dz


def candidates_per_cell(n_valid, spc):
    v = np.arange(n_valid, dtype=np.float64)
    return (np.floor((v + 1) * spc) - np.floor(v * spc)).astype(np.int64)


def random_index_samples(n, phi, spc, seed, chunk=1 << 22):
    """yields (q, keep) per chunk of candidates, in candidate order: q the index-space candidates, keep where phi(q) < 0"""
    valid = valid_cells(n, phi)
    owner = np.repeat(valid, candidates_per_cell(len(valid), spc))
    key = (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    for j0 in range(0, len(owner), chunk):
        ids = owner[j0:j0 + chunk]
        j = np.arange(j0, j0 + len(ids), dtype=np.uint64)
        ctr = np.zeros((len(ids), 4), np.uint32)
        ctr[:, 0], ctr[:, 1] = (j & _MASK).astype(np.uint32), (j >> np.uint64(32)).astype(np.uint32)
        w = philox4x32_10(ctr, key)
        cell = np.stack([ids % (n[0] - 1), (ids // (n[0] - 1)) % (n[1] - 1), ids // ((n[0] - 1) * (n[1] - 1))], 1).astype(np.float64)
        q = cell + (w[:, :3] >> np.uint32(8)).astype(np.float64) * 2.0 ** -24
        yield q, trilinear(n, phi, q[:, 0], q[:, 1], q[:, 2]) < 0


def random_spc(n, h, domain_bits, offset, span, ppc):
    c, _, _ = node_box(n, h, offset, span)
    r = c / (1.0 / (1 << domain_bits))
    return c, float(ppc) * (r * r * r)


def sample_random(n, h, phi, domain_bits, offset, span, ppc, seed):
    c, spc = random_spc(n, h, domain_bits, offset, span, ppc)
    out = [(np.asarray(offset, np.float64) + q[keep] * c).astype(np.float32) for q, keep in random_index_samples(n, phi, spc, seed)]
    return np.concatenate(out, 0) if out else np.zeros((0, 3), np.float32)


def sample_lattice(n, h, phi, domain_bits, offset, span, ppc, x_slabs=None):
    """x_slabs: optional (lo, hi) of simulation-cell x indices to restrict to (rows of those slabs, in order)."""
    k = round(ppc ** (1 / 3))
    assert k ** 3 == ppc and 1 <= k <= 4
    c, lo_w, hi_w = node_box(n, h, offset, span)
    dx = 1.0 / (1 << domain_bits)
    cells = 1 << domain_bits
    lo = [max(0, int(np.floor(lo_w[d] / dx)) - 1) for d in range(3)]
    hi = [min(cells, int(np.ceil(hi_w[d] / dx)) + 2) for d in range(3)]
    a = (np.arange(k, dtype=np.float64) - (k - 1) * 0.5) / k
    offs = np.stack(np.meshgrid(a, a, a, indexing="ij"), -1).reshape(-1, 3)
    off = np.asarray(offset, np.float64)
    xs = range(lo[0], hi[0]) if x_slabs is None else range(max(lo[0], x_slabs[0]), min(hi[0], x_slabs[1]))
    out = []
    for i in xs:
        j, kk = np.meshgrid(np.arange(lo[1], hi[1]), np.arange(lo[2], hi[2]), indexing="ij")
        cl = np.stack([np.full_like(j, i), j, kk], -1).reshape(-1, 1, 3).astype(np.float64)
        x = ((cl + offs[None]) * dx).reshape(-1, 3).astype(np.float32)
        q = (x.astype(np.float64) - off) / c
        inside = np.all((q >= 0) & (q <= np.asarray(n, np.float64) - 1), 1)
        keep = np.zeros(len(x), bool)
        if inside.any():
            qi = q[inside]
            keep[inside] = trilinear(n, phi, qi[:, 0], qi[:, 1], qi[:, 2]) < 0
        if keep.any():
            out.append(x[keep])
    return np.concatenate(out, 0) if out else np.zeros((0, 3), np.float32)


# ---- synthetic level sets: (n, h, phi[k, j, i] float32) ---------------------------------------------------------------------------
def _grid(n, h):
    k, j, i = np.meshgrid(np.arange(n[2]), np.arange(n[1]), np.arange(n[0]), indexing="ij")
    return i * h, j * h, k * h


def sphere(n, h, center, radius):
    x, y, z = _grid(n, h)
    return n, h, (np.sqrt((x - center[0]) ** 2 + (y - center[1]) ** 2 + (z - center[2]) ** 2) - radius).astype(np.float32)


def torus(n, h, center, R, r):
    x, y, z = _grid(n, h)
    q = np.sqrt((x - center[0]) ** 2 + (z - center[2]) ** 2) - R
    return n, h, (np.sqrt(q ** 2 + (y - center[1]) ** 2) - r).astype(np.float32)


def box(n, h, lo, hi):
    x, y, z = _grid(n, h)
    d = np.maximum.reduce([lo[0] - x, x - hi[0], lo[1] - y, y - hi[1], lo[2] - z, z - hi[2]])
    return n, h, d.astype(np.float32)


def plate(n, h, k0):
    """one level-set cell thick: negative only on the node layers k0 and k0 + 1 (inside 1 < i, j < n - 2)"""
    phi = np.ones((n[2], n[1], n[0]), np.float32)
    phi[k0:k0 + 2, 1:-1, 1:-1] = -0.5
    return n, h, phi


def two_bodies(n, h):
    _, _, a = sphere(n, h, (0.3 * (n[0] - 1) * h, 0.5 * (n[1] - 1) * h, 0.5 * (n[2] - 1) * h), 0.2 * (n[0] - 1) * h)
    _, _, b = sphere(n, h, (0.75 * (n[0] - 1) * h, 0.5 * (n[1] - 1) * h, 0.5 * (n[2] - 1) * h), 0.15 * (n[0] - 1) * h)
    return n, h, np.minimum(a, b)


def all_negative(n, h):
    return n, h, np.full((n[2], n[1], n[0]), -1.0, np.float32)


def dragonish(n=(12, 18, 60), h=0.25):
    """two_dragons.sdf's proportions (77 x 118 x 401 nodes) at small size: two blobs along z"""
    x, y, z = _grid(n, h)
    L = [(n[d] - 1) * h for d in range(3)]
    a = np.sqrt(((x - 0.5 * L[0]) / (0.4 * L[0])) ** 2 + ((y - 0.45 * L[1]) / (0.4 * L[1])) ** 2 + ((z - 0.25 * L[2]) / (0.2 * L[2])) ** 2) - 1
    b = np.sqrt(((x - 0.5 * L[0]) / (0.35 * L[0])) ** 2 + ((y - 0.55 * L[1]) / (0.4 * L[1])) ** 2 + ((z - 0.72 * L[2]) / (0.22 * L[2])) ** 2) - 1
    return n, h, (np.minimum(a, b) * min(L) * 0.2).astype(np.float32)
