"""Mesh level sets without a GPU (claymore_b200.mesh, DESIGN.md section 2.12): the C ABI's structs and exports, the OBJ parser with
SDFGen's loader quirks M1-M8 fixed, the host-only header of cb200_mesh_levelset and its rejections, the scene front-end's errors,
and the SDFGen goldens themselves, against the live SDFGen shim and against an independent float64 restatement."""
import ctypes as C
import glob
import json
import os
import subprocess

import numpy as np
import pytest

import mesh_cases as M
from claymore_b200 import _capi, mesh, scene, sdf

GOLDENS = sorted(glob.glob(os.path.join(M.GOLDEN, "ref_sdfgen_*.npz")))
HEADER = os.path.join(M.ROOT, "include", "claymore_b200.h")


def test_struct_layouts_match_gcc(tmp_path):
    src = tmp_path / "l.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "claymore_b200.h"\nint main(void){\n'
                   'printf("%zu %zu %zu %zu %zu\\n", sizeof(cb200_mesh_header), offsetof(cb200_mesh_header, nt), offsetof(cb200_mesh_header, min), offsetof(cb200_mesh_header, max), 0);\n'
                   'printf("%zu %zu %zu\\n", sizeof(cb200_mesh_levelset_params), offsetof(cb200_mesh_levelset_params, padding), offsetof(cb200_mesh_levelset_params, exact_band));\n'
                   'return 0;}\n')
    subprocess.check_call(["gcc", "-I", os.path.dirname(HEADER), "-o", str(tmp_path / "l"), str(src)])
    out = subprocess.check_output([str(tmp_path / "l")]).decode().split("\n")
    H, P = _capi.MeshHeader, _capi.MeshLevelSetParams
    assert out[0].split() == [str(x) for x in (C.sizeof(H), H.nt.offset, H.min.offset, H.max.offset, 0)]
    assert out[1].split() == [str(x) for x in (C.sizeof(P), P.padding.offset, P.exact_band.offset)]


def test_exports():
    L = _capi.lib()
    for name in ("cb200_obj_parse", "cb200_mesh_levelset"):
        assert hasattr(L, name)


@pytest.mark.parametrize("text", [
    "v 1 2\n", "v 1 2 x\n", "v 1 2 inf\n", "v 1 nan 2\n", "v 0 0 0\nv 1 0 0\nv 0 1 0\nf 1 2\n", "v 0 0 0\nv 1 0 0\nv 0 1 0\nf 1 2 4\n",
    "v 0 0 0\nv 1 0 0\nv 0 1 0\nf 0 1 2\n", "v 0 0 0\nv 1 0 0\nv 0 1 0\nf 1 2 x\n", "v 0 0 0\nv 1 0 0\nv 0 1 0\nf -4 -1 -2\n",
    "v 0 0 0\nv 1 0 0\nv 0 1 0\nf 1 2 3.5\n", "v 0 0 0\nv 1 0 0\nv 0 1 0\nf 1 2 99999999999999999999\n"])
def test_parser_rejects(text):
    with pytest.raises(ValueError):
        mesh.parse_obj(text)


TRI = "v 0 0 0\nv 1 0 0\nv 0 1 0\n"


def test_m1_only_v_lines_are_vertices():
    m = mesh.parse_obj("vt 5 5\nvp 9 9 9\n" + TRI + "f 1 2 3\n")
    assert m.vertices.shape == (3, 3) and m.vertices.max() == 1 and m.triangles.tolist() == [[0, 1, 2]]


def test_m2_vn_lines_are_ignored():
    assert mesh.parse_obj(TRI + "vn 0 0 1\nf 1 2 3\n").triangles.tolist() == [[0, 1, 2]]


def test_m3_slashed_references():
    m = mesh.parse_obj(TRI + "vt 0 0\nvn 0 0 1\nf 1/1/1 2//1 3/1\n")
    assert m.triangles.tolist() == [[0, 1, 2]]


def test_m4_polygons_become_fans():
    m = mesh.parse_obj(TRI + "v 1 1 0\nv 2 2 0\nf 1 2 4 5 3\n")
    assert m.triangles.tolist() == [[0, 1, 3], [0, 3, 4], [0, 4, 2]]


def test_m5_negative_references():
    m = mesh.parse_obj(TRI + "f -3 -2 -1\nv 5 5 5\nf -4 -1 -2\n")
    assert m.triangles.tolist() == [[0, 1, 2], [0, 3, 2]]


def test_m6_out_of_range_is_rejected():
    with pytest.raises(ValueError):
        mesh.parse_obj(TRI + "f 1 2 4\n")


def test_m7_write_round_trips_bitwise(tmp_path):
    g = M.golden(GOLDENS[0])
    hdr = _capi.SdfHeader()
    hdr.ni, hdr.nj, hdr.nk = (int(x) for x in g["dims"])
    hdr.min[:] = [float(x) for x in g["origin"]]
    hdr.h = float(g["h"])
    phi = g["phi"].copy()
    phi[:3] = [-0.0, np.float32(1e-38), np.float32(3.4e38)]
    ls = sdf.LevelSet(hdr, phi)
    sdf.write(ls, str(tmp_path / "a.sdf"))
    back = sdf.read(str(tmp_path / "a.sdf"))
    assert back.n == ls.n and np.array_equal(np.asarray(back.header.min[:], np.float32), g["origin"]) and back.h == ls.h
    assert np.array_equal(back.phi.view(np.uint32), phi.view(np.uint32))


def test_m8_box_counts_every_vertex():
    """SDFGen's `else if` never lets the first vertex raise the max: on the torus (its first vertex has the largest x) main's lattice
    has one node fewer in x at h = 0.035; here the box is the true one"""
    v, t = M.torus()
    m = mesh.Mesh(v, t)
    assert mesh.header(m, 0.035).ni == M.header(v, 0.035, 1)[0][0] == 59
    assert M.header(v, 0.035, 1, M.sdfgen_box(v))[0][0] == 58


def test_torus_parse_equals_arrays():
    v, t = M.torus()
    text = ("# a comment\ng torus\n" + M.plain_obj(v, t)).encode()
    m = mesh.parse_obj(text)
    assert np.array_equal(m.vertices.view(np.uint32), v.view(np.uint32)) and np.array_equal(m.triangles, t)
    hdr = _capi.MeshHeader()
    assert _capi.lib().cb200_obj_parse(text, len(text), C.byref(hdr), None, None, 0, 0) == 0
    assert (hdr.nv, hdr.nt) == (5205, 10410)
    assert np.array_equal(np.asarray(hdr.min[:], np.float32), v.min(0)) and np.array_equal(np.asarray(hdr.max[:], np.float32), v.max(0))


def test_parse_capacity_too_small():
    hdr = _capi.MeshHeader()
    text = (TRI + "f 1 2 3\n").encode()
    buf = np.empty(9, np.float32)
    tri = np.empty(3, np.int32)
    assert _capi.lib().cb200_obj_parse(text, len(text), C.byref(hdr), buf.ctypes.data, tri.ctypes.data, 2, 1) != 0
    assert _capi.lib().cb200_obj_parse(text, len(text), C.byref(hdr), buf.ctypes.data, tri.ctypes.data, 3, 0) != 0


@pytest.mark.parametrize("name", ["cube_on_nodes", "two_bodies", "unreferenced", "floor"])
@pytest.mark.parametrize("h,padding", [(0.05, 1), (0.031, 3), (0.1, 0), (0.07, 2)])
def test_header_equals_sdfgen_main(name, h, padding):
    if M.shim() is None:
        pytest.skip("oracle/_ref/libclaymore_ref_sdfgen.so not built (oracle/build_ref_sdfgen.sh)")
    v, t = M.cases()[name][:2]
    hdr = mesh.header(mesh.Mesh(v, t), h, padding)
    dims, org, htok, _ = M.ref_main(M.plain_obj(v, t), h, padding)
    assert [hdr.ni, hdr.nj, hdr.nk] == dims
    assert org == ["%g" % x for x in np.asarray(hdr.min[:], np.float32)] and htok == "%g" % np.float32(h)


def _levelset_err(v, t, h=0.1, padding=1, band=1, cap=None):
    hdr = _capi.SdfHeader()
    p = _capi.MeshLevelSetParams(h, padding, band)
    v = np.ascontiguousarray(v, np.float32)
    t = np.ascontiguousarray(t, np.int32)
    phi = np.empty(max(cap or 0, 1), np.float32)
    return _capi.lib().cb200_mesh_levelset(v.ctypes.data, len(v), t.ctypes.data, len(t), C.byref(p), C.byref(hdr),
                                           phi.ctypes.data if cap is not None else None, cap or 0, None)


def test_levelset_rejections_before_device_work():
    v, t = M.cube()
    assert _levelset_err(v, t) == 0
    inv = 1  # cudaErrorInvalidValue
    for kw in (dict(h=0.0), dict(h=-1.0), dict(h=float("inf")), dict(h=float("nan")), dict(band=-1), dict(band=9), dict(h=1e-4),
               dict(cap=10)):
        assert _levelset_err(v, t, **kw) == inv, kw
    assert _levelset_err(v, t[:0]) == inv
    assert _levelset_err(v, np.vstack([t, [[0, 1, 8]]])) == inv
    assert _levelset_err(v, np.vstack([t, [[0, -1, 2]]])) == inv
    bad = v.copy()
    bad[3, 1] = np.inf
    assert _levelset_err(bad, t) == inv
    flat = v.copy()
    flat[:, 2] = 0   # a flat mesh still has 2 * padding cells across
    assert _levelset_err(flat, t) == 0
    with pytest.raises(ValueError):
        mesh.header(mesh.Mesh(v, t), 1e-4)


def test_padding_below_one_is_one():
    v, t = M.cube()
    a, b = mesh.header(mesh.Mesh(v, t), 0.1, 1), mesh.header(mesh.Mesh(v, t), 0.1, -5)
    assert (a.ni, a.nj, a.nk, a.min[0]) == (b.ni, b.nj, b.nk, b.min[0])


def _doc(**kw):
    d = {"simulation": {"frames": 2}, "models": [{"constitutive": "jfluid", "file": "box", "offset": [0.4, 0.4, 0.4], "span": [0.1, 0.1, 0.1]}]}
    d.update(kw)
    return d


def test_scene_errors_before_any_simulator(tmp_path, monkeypatch):
    import claymore_b200.simulator as S
    monkeypatch.setattr(S.GmpmSimulator, "__init__", lambda *a, **k: pytest.fail("a simulator was created"))
    v, t = M.cube()
    (tmp_path / "c.obj").write_text(M.plain_obj(v, t))
    (tmp_path / "bad.obj").write_text("v 0 0 0\nf 1 2 3\n")
    base = {"offset": [0.3, 0.3, 0.3], "span": [0.2, 0.2, 0.2]}
    bad = [
        _doc(models=[{"constitutive": "jfluid", "file": "bad.obj", **base}]),
        _doc(models=[{"constitutive": "jfluid", "file": "missing.obj", **base}]),
        _doc(models=[{"constitutive": "jfluid", "file": "c.obj", "h": 0, **base}]),
        _doc(models=[{"constitutive": "jfluid", "file": "c.obj", "exact_band": 9, **base}]),
        _doc(models=[{"constitutive": "jfluid", "file": "c.obj", "offset": [0.9, 0.3, 0.3], "span": [0.2, 0.2, 0.2]}]),
        _doc(boundaries=[{"shape": "levelset", "file": "bad.obj", **base}]),
        _doc(boundaries=[{"shape": "levelset", "file": "c.obj", "padding": "x", **base}]),
        _doc(boundaries=[{"shape": "levelset", "file": "c.stl", **base}]),
        _doc(sinks=[{"shape": "levelset", "file": "c.obj", "h": -1.0, **base}]),
    ]
    for i, d in enumerate(bad):
        p = tmp_path / f"s{i}.json"
        p.write_text(json.dumps(d))
        with pytest.raises(ValueError) as e:
            scene.parse_scene(str(p))
        if i == 7:
            assert "must name an .sdf" in str(e.value)


@pytest.mark.parametrize("path", GOLDENS, ids=lambda p: os.path.basename(p))
def test_goldens_equal_live_sdfgen(path):
    L = M.shim()
    if L is None:
        pytest.skip("oracle/_ref/libclaymore_ref_sdfgen.so not built (oracle/build_ref_sdfgen.sh)")
    g = M.golden(path)
    n, lo, phi = M.ref_level_set(L, g["vertices"], g["triangles"], float(g["h"]), int(g["padding"]), int(g["exact_band"]))
    assert n == list(g["dims"]) and np.array_equal(lo, g["origin"]) and np.array_equal(phi.view(np.uint32), g["phi"].view(np.uint32))


def _nodes(g):
    n = [int(x) for x in g["dims"]]
    h = np.float32(g["h"])
    k, j, i = np.meshgrid(np.arange(n[2]), np.arange(n[1]), np.arange(n[0]), indexing="ij")
    idx = np.stack([i.ravel(), j.ravel(), k.ravel()], 1)
    x = (idx.astype(np.float32) * h + g["origin"].astype(np.float32)).astype(np.float64)
    return x


def _point_triangle_min(x, v, t):
    """float64 distance from every point x to the nearest triangle (closest point by clamped barycentrics, Ericson's method)"""
    a, b, c = v[t[:, 0]], v[t[:, 1]], v[t[:, 2]]
    best = np.full(len(x), np.inf)
    for s in range(0, len(t), 256):
        A, B, Cc = a[s:s + 256][None], b[s:s + 256][None], c[s:s + 256][None]
        P = x[:, None]
        ab, ac, ap = B - A, Cc - A, P - A
        d1, d2 = (ab * ap).sum(-1), (ac * ap).sum(-1)
        bp, cp = P - B, P - Cc
        d3, d4 = (ab * bp).sum(-1), (ac * bp).sum(-1)
        d5, d6 = (ab * cp).sum(-1), (ac * cp).sum(-1)
        va, vb, vc = d3 * d6 - d5 * d4, d5 * d2 - d1 * d6, d1 * d4 - d3 * d2
        with np.errstate(all="ignore"):
            denom = va + vb + vc
            vv, ww = np.where(denom != 0, vb / denom, 0), np.where(denom != 0, vc / denom, 0)
            q = A + ab * vv[..., None] + ac * ww[..., None]
            # edges and vertices
            cands = [q]
            for E0, E1 in ((A, B), (A, Cc), (B, Cc)):
                e = E1 - E0
                tt = np.clip(((P - E0) * e).sum(-1) / np.maximum((e * e).sum(-1), 1e-300), 0, 1)
                cands.append(E0 + e * tt[..., None])
        inside = (va >= 0) & (vb >= 0) & (vc >= 0) & (denom > 0)
        dq = np.where(inside, np.linalg.norm(P - q, axis=-1), np.inf)
        de = np.min([np.linalg.norm(P - c_, axis=-1) for c_ in cands[1:]], axis=0)
        best = np.minimum(best, np.minimum(dq, de).min(axis=1))
    return best


def test_golden_band_distances_float64():
    """nodes within the exact band of the nearest triangle: |phi| is the float64 point-triangle minimum within float rounding"""
    for name in ("torus_h07_p1_b1", "degenerate", "two_bodies", "single_triangle"):
        g = M.golden(os.path.join(M.GOLDEN, f"ref_sdfgen_{name}.npz"))
        x = _nodes(g)
        v, t = g["vertices"].astype(np.float64), g["triangles"]
        area = np.linalg.norm(np.cross(v[t[:, 1]] - v[t[:, 0]], v[t[:, 2]] - v[t[:, 0]]), axis=1)
        t = t[area > 0]
        rng = np.random.default_rng(0)
        sel = rng.choice(len(x), min(len(x), 1500), replace=False)
        d = _point_triangle_min(x[sel], v, t)
        near = d < float(g["h"]) * 0.9   # inside every triangle's band box that decides it
        phi = np.abs(g["phi"][sel].astype(np.float64))
        assert near.sum() > 20, name
        err = np.abs(phi[near] - d[near])
        assert err.max() <= 1e-5 * (1 + np.abs(v).max()), (name, err.max())


def test_golden_torus_sign_equals_winding_number():
    g = M.golden(os.path.join(M.GOLDEN, "ref_sdfgen_torus_h055_p3_b1.npz"))
    x = _nodes(g)
    phi = g["phi"]
    rng = np.random.default_rng(1)
    cand = np.flatnonzero(np.abs(phi) > 1e-3 * float(g["h"]))
    sel = rng.choice(cand, 800, replace=False)
    v, t = g["vertices"].astype(np.float64), g["triangles"]
    a, b, c = v[t[:, 0]][None] - x[sel][:, None], v[t[:, 1]][None] - x[sel][:, None], v[t[:, 2]][None] - x[sel][:, None]
    la, lb, lc = (np.linalg.norm(q, axis=-1) for q in (a, b, c))
    num = np.einsum("pti,pti->pt", a, np.cross(b, c))
    den = la * lb * lc + np.einsum("pti,pti->pt", a, b) * lc + np.einsum("pti,pti->pt", b, c) * la + np.einsum("pti,pti->pt", c, a) * lb
    w = np.abs(np.arctan2(num, den).sum(axis=1)) / (2 * np.pi)
    assert np.array_equal(w > 0.5, phi[sel] < 0)
