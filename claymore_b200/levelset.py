"""Analytic signed-distance fields for the collider (GmpmSimulator.set_collider).

Each generator samples a shape on the (4G)^3 grid nodes x = index * dx and returns (sdf, grad): the signed distance as a
float32 array of shape (N, N, N) and its gradient as float32 (3, N, N, N), both row-major over the nodes like the reference's
`<name>_sdf.bin` / `_grad_{0,1,2}.bin` files (Projects/MGSP/boundary_condition.cuh:297-320).  Inside is negative.
"""
import os

import numpy as np


def _sample(cfg, fn):
    """fn(x, Y, Z) -> (sdf, [gx, gy, gz]) on one x slab of the node lattice (float64, broadcastable to (N, N)); slab by slab so
    that a 512^3 field (2 GiB in float32) needs no float64 copy of itself."""
    n = 4 * cfg.grid_size
    y = np.arange(n, dtype=np.float64) * cfg.dx
    Y, Z = np.meshgrid(y, y, indexing="ij")
    sdf = np.empty((n, n, n), np.float32)
    grad = np.empty((3, n, n, n), np.float32)
    for i in range(n):
        d, g = fn(i * cfg.dx, Y, Z)
        sdf[i] = d
        for c in range(3):
            grad[c, i] = g[c]
    return sdf, grad


def box(cfg, lo, hi):
    """Axis-aligned box [lo, hi] (world units)."""
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    c, h = (lo + hi) / 2, (hi - lo) / 2

    def fn(x, Y, Z):
        p = [np.full_like(Y, x - c[0]), Y - c[1], Z - c[2]]
        q = [np.abs(p[i]) - h[i] for i in range(3)]
        s = [np.where(p[i] < 0, -1.0, 1.0) for i in range(3)]
        o = [np.maximum(q[i], 0.0) for i in range(3)]
        outside = np.sqrt(o[0] ** 2 + o[1] ** 2 + o[2] ** 2)
        sdf = outside + np.minimum(np.maximum(q[0], np.maximum(q[1], q[2])), 0.0)
        axis = np.argmax(np.stack(q), axis=0)   # inside: the nearest face
        safe = np.where(outside > 0, outside, 1.0)
        return sdf, [np.where(outside > 0, o[i] / safe * s[i], np.where(axis == i, s[i], 0.0)) for i in range(3)]
    return _sample(cfg, fn)


def sphere(cfg, center, radius):
    def fn(x, Y, Z):
        p = [np.full_like(Y, x - center[0]), Y - center[1], Z - center[2]]
        r = np.sqrt(p[0] ** 2 + p[1] ** 2 + p[2] ** 2)
        safe = np.where(r > 0, r, 1.0)
        return r - radius, [np.where(r > 0, p[i] / safe, 0.0) for i in range(3)]
    return _sample(cfg, fn)


def plane(cfg, point, normal):
    """Half-space behind the plane through `point`: the solid is where (x - point) . normal < 0."""
    u = np.asarray(normal, np.float64)
    u = u / np.linalg.norm(u)

    def fn(x, Y, Z):
        return (x - point[0]) * u[0] + (Y - point[1]) * u[1] + (Z - point[2]) * u[2], [u[0], u[1], u[2]]
    return _sample(cfg, fn)


def load(cfg, prefix):
    """The reference's file form: <prefix>_sdf.bin and <prefix>_grad_{0,1,2}.bin, float32, (4G)^3 each."""
    n = 4 * cfg.grid_size

    def read(suffix):
        a = np.fromfile(prefix + suffix, dtype=np.float32)
        if a.size != n ** 3:
            raise ValueError(f"{prefix + suffix}: {a.size} floats, expected {n ** 3} for a {n}^3 node grid")
        return a.reshape(n, n, n)
    if not os.path.exists(prefix + "_sdf.bin"):
        raise FileNotFoundError(prefix + "_sdf.bin")
    return read("_sdf.bin"), np.stack([read(f"_grad_{d}.bin") for d in range(3)])
