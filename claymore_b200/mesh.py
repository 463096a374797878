"""Level sets from triangle meshes: SDFGen's make_level_set3 (Externals/SDFGen/makelevelset3.cpp) on the device, bit for bit.

    mesh = mesh.read_obj("dragon.obj")                        # Wavefront OBJ, with SDFGen's loader quirks M1-M8 fixed (DESIGN §2.12)
    ls = mesh.levelset(mesh, h=0.01, padding=1)               # an sdf.LevelSet, as sdf.read would return for SDFGen's output
    sim.init_model_sdf(material, ls, offset, span, v0)        # every .sdf consumer takes it unchanged

The lattice is SDFGen's: node 0 at the vertex box minus padding h, (max - min) / h nodes per axis (truncated), distances exact within
exact_band cells of each triangle and from fast sweeping beyond, negative inside by the parity of crossings along +x (a mesh that
is not watertight gives streaks of wrong sign).
"""
import ctypes as C

import numpy as np

from . import sdf
from ._capi import MeshHeader, MeshLevelSetParams, SdfHeader, check, lib


class Mesh:
    """A triangle mesh: vertices (n, 3) float32 and triangles (m, 3) int32, 0-based."""

    def __init__(self, vertices, triangles):
        self.vertices = np.ascontiguousarray(vertices, dtype=np.float32).reshape(-1, 3)
        self.triangles = np.ascontiguousarray(triangles, dtype=np.int32).reshape(-1, 3)

    @property
    def bounds(self):
        """(lo, hi): the vertex bounding box, float32."""
        return self.vertices.min(axis=0), self.vertices.max(axis=0)


def parse_obj(text):
    """Parses Wavefront OBJ text (bytes or str) with cb200_obj_parse.  Raises ValueError for anything it rejects."""
    if isinstance(text, str):
        text = text.encode()
    hdr = MeshHeader()
    if lib().cb200_obj_parse(text, len(text), C.byref(hdr), None, None, 0, 0) != 0:
        raise ValueError("not a valid .obj mesh (`v` lines need three finite numbers, `f` lines three or more vertex references "
                         "that are non-zero integers within the vertices)")
    v = np.empty((hdr.nv, 3), np.float32)
    t = np.empty((hdr.nt, 3), np.int32)
    check(lib().cb200_obj_parse(text, len(text), C.byref(hdr), v.ctypes.data_as(C.c_void_p), t.ctypes.data_as(C.c_void_p), hdr.nv, hdr.nt),
          "obj_parse")
    return Mesh(v, t)


def read_obj(path):
    with open(path, "rb") as f:
        return parse_obj(f.read())


def _params(h, padding, exact_band):
    p = MeshLevelSetParams()
    p.h, p.padding, p.exact_band = float(h), int(padding), int(exact_band)
    return p


def _call(mesh, h, padding, exact_band, phi=None, stream=None):
    hdr = SdfHeader()
    x, t = mesh.vertices, mesh.triangles
    out = phi.ctypes.data_as(C.c_void_p) if phi is not None else None
    return hdr, lib().cb200_mesh_levelset(x.ctypes.data_as(C.c_void_p), len(x), t.ctypes.data_as(C.c_void_p), len(t),
                                          C.byref(_params(h, padding, exact_band)), C.byref(hdr), out,
                                          0 if phi is None else phi.size, C.c_void_p(stream) if stream else None)


def header(mesh, h, padding=1, exact_band=1):
    """The SdfHeader of mesh's level set (host only, no device work).  ValueError for what cb200_mesh_levelset rejects."""
    hdr, err = _call(mesh, h, padding, exact_band)
    if err != 0:
        raise ValueError(f"no level set for this mesh at h={h!r}, padding={padding!r}, exact_band={exact_band!r} (h finite and > 0, "
                         "exact_band in 0..8, at least one triangle, finite vertices, 2 or more nodes per axis and fewer than 2^31)")
    return hdr


def levelset(mesh, h, padding=1, exact_band=1, stream=None):
    """The signed distance level set of `mesh` on the current device, as an sdf.LevelSet (SDFGen's header and phi, i fastest)."""
    hdr = header(mesh, h, padding, exact_band)
    phi = np.empty(hdr.ni * hdr.nj * hdr.nk, np.float32)
    hdr, err = _call(mesh, h, padding, exact_band, phi, stream)
    check(err, "mesh_levelset")
    return sdf.LevelSet(hdr, phi)


__all__ = ["Mesh", "parse_obj", "read_obj", "header", "levelset"]
