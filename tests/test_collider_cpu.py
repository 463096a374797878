"""CPU tests of the signed-distance collider (SignedDistanceGrid, Projects/MGSP/boundary_condition.cuh).

The oracle's restatement (oracle/collider_oracle.c: orc_collider_resolve) is pinned bit for bit against the reference's own
detect_and_resolve_collision compiled for the host (oracle/_ref/libclaymore_ref_collider.so, built by oracle/build_ref.sh
where the reference checkout exists); the two fixed quirks are asserted instead where they apply.  Then oracle physics, and
the C ABI / adapter surface."""
import ctypes as C
import os
import re
import shutil
import subprocess
import zlib

import numpy as np
import pytest

import collider_oracle_binding as cob
import oracle_binding as ob
from claymore_b200 import levelset
from claymore_b200._capi import Config as EngineConfig

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libclaymore_ref_collider.so")
REFERENCE = os.environ.get("CLAYMORE_REFERENCE", "/root/reference")


def _ref():
    if not os.path.exists(REF_LIB):
        pytest.skip("reference collider not built (oracle/build_ref.sh needs the reference checkout)")
    L = C.CDLL(REF_LIB)
    L.ref_collider_resolve.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_float, C.c_void_p]
    return L


def _cfg(L):
    return ob.make_config(domain_bits=L.ref_collider_domain_bits(), boundary=L.ref_collider_boundary())


def _rot(ax, ay, az):
    cx, sx, cy, sy, cz, sz = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay), np.cos(az), np.sin(az)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rx @ Ry @ Rz


def _field(cfg, shape):
    ecfg = EngineConfig(domain_bits=cfg.domain_bits, boundary=cfg.boundary)
    if shape == "sphere":
        return levelset.sphere(ecfg, (0.52, 0.47, 0.5), 0.21)
    return levelset.box(ecfg, (0.3, 0.28, 0.33), (0.68, 0.61, 0.7))


def _params(rot, trans, trans_vel, omega, dsdt, scale, friction, typ):
    return np.array(list(np.asarray(rot, np.float32).reshape(9)) + list(trans) + list(trans_vel) + list(omega) + [dsdt, scale, friction, typ], np.float32)


def _collider(p):
    col = cob.Collider()
    col.rot_mat[:] = [float(v) for v in p[:9]]
    col.trans[:], col.trans_vel[:], col.omega[:] = [float(v) for v in p[9:12]], [float(v) for v in p[12:15]], [float(v) for v in p[15:18]]
    col.dsdt, col.scale, col.friction, col.type = float(p[18]), float(p[19]), float(p[20]), int(p[21])
    return col


def _block_field(cfg, sdf, grad):
    """the oracle's layout of the field: G^3 blocks x [4][64]"""
    n = 4 * (1 << (cfg.domain_bits - 2))
    g = n // 4
    a = np.concatenate([sdf[None], grad]).reshape(4, g, 4, g, 4, g, 4)
    return np.ascontiguousarray(a.transpose(1, 3, 5, 0, 2, 4, 6).reshape(-1)).astype(np.float32)


def _run_both(L, cfg, sdf, grad, p, t, nodes, vel):
    field_nodes = np.ascontiguousarray(np.concatenate([sdf.reshape(1, -1), grad.reshape(3, -1)]), np.float32)
    bc = np.ascontiguousarray(np.concatenate([nodes >> 2, nodes & 3], 1).astype(np.int32))
    vr = np.ascontiguousarray(vel.copy(), np.float32)
    L.ref_collider_resolve(ob.ptr(field_nodes), ob.ptr(p), len(nodes), ob.ptr(bc), t, ob.ptr(vr))
    blocks = _block_field(cfg, sdf, grad)
    col = _collider(p)
    col.sdf = blocks.ctypes.data
    vo = np.ascontiguousarray(vel.copy(), np.float32)
    lib = cob.lib()
    for i in range(len(nodes)):
        nd = np.ascontiguousarray(nodes[i], np.int32)
        lib.orc_collider_resolve(C.byref(cfg), C.byref(col), t, ob.ptr(nd), ob.ptr(vo[i]))
    return vr, vo


def _queries(cfg, rng, n=1500):
    N = 4 * (1 << (cfg.domain_bits - 2))
    nodes = rng.integers(0, N, size=(n, 3)).astype(np.int32)   # includes the wall band
    vel = rng.normal(0, 1.0, size=(n, 3)).astype(np.float32)
    return nodes, vel


MOTIONS = {
    "static": dict(),
    "trans": dict(trans=(0.03, -0.02, 0.01)),
    "trans_vel": dict(trans_vel=(0.4, -0.3, 0.2)),
    "scale": dict(scale=1.15),
    "dsdt": dict(dsdt=0.6),
    "rot_mat": dict(rot=_rot(0.3, -0.2, 0.5)),
}


@pytest.mark.parametrize("shape", ["sphere", "box"])
@pytest.mark.parametrize("motion", sorted(MOTIONS))
@pytest.mark.parametrize("typ", [0, 1, 2])
@pytest.mark.parametrize("friction", [0.0, 0.3])
@pytest.mark.parametrize("t", [0.0, 0.37])
def test_resolve_matches_reference_bit_for_bit(shape, motion, typ, friction, t):
    """omega = 0: the oracle's resolve equals the reference's, bit for bit, on every queried node (wall band included)."""
    L = _ref()
    cfg = _cfg(L)
    m = MOTIONS[motion]
    p = _params(m.get("rot", np.eye(3)), m.get("trans", (0, 0, 0)), m.get("trans_vel", (0, 0, 0)), (0, 0, 0), m.get("dsdt", 0.0), m.get("scale", 1.0), friction, typ)
    sdf, grad = _field(cfg, shape)
    rng = np.random.default_rng(zlib.crc32(f"{shape}-{motion}-{typ}-{friction}-{t}".encode()))
    nodes, vel = _queries(cfg, rng, n=3000)
    vr, vo = _run_both(L, cfg, sdf, grad, p, np.float32(t), nodes, vel)
    assert np.isfinite(vr).all()
    assert np.array_equal(vr.view(np.uint32), vo.view(np.uint32))
    changed = (vr != vel).any(1)
    assert changed.sum() > 10, "the queries must hit the object"


def test_wall_band_reports_no_hit():
    """query_sdf reports no hit inside the wall band (kept): a field that is solid everywhere leaves band nodes untouched."""
    L = _ref()
    cfg = _cfg(L)
    N = 4 * (1 << (cfg.domain_bits - 2))
    sdf = -np.ones((N, N, N), np.float32)
    grad = np.zeros((3, N, N, N), np.float32)
    grad[1] = 1.0
    p = _params(np.eye(3), (0, 0, 0), (0, 0, 0), (0, 0, 0), 0.0, 1.0, 0.0, 0)
    nodes, vel = _queries(cfg, np.random.default_rng(3))
    vr, vo = _run_both(L, cfg, sdf, grad, p, np.float32(0.0), nodes, vel)
    lo, hi = 4 * cfg.boundary, N - 4 * cfg.boundary
    band = ((nodes < lo) | (nodes >= hi)).any(1)
    assert band.any() and (~band).any()
    assert np.array_equal(vo[band], vel[band]) and np.array_equal(vr[band], vel[band])
    assert (vo[~band] == 0).all()


@pytest.mark.parametrize("friction", [0.0, 0.3])
def test_zero_gradient_normal_is_fixed(friction):
    """Inside a region whose interpolated gradient is 0 the reference normalises 0/0: SLIP writes NaN and SEPARATE can never take its
    zero-normal branch.  Here SLIP leaves the velocity unchanged and SEPARATE zeroes it; STICKY stays bit-exact."""
    L = _ref()
    cfg = _cfg(L)
    N = 4 * (1 << (cfg.domain_bits - 2))
    sdf = -np.ones((N, N, N), np.float32)
    grad = np.zeros((3, N, N, N), np.float32)
    lo, hi = 4 * cfg.boundary, N - 4 * cfg.boundary
    rng = np.random.default_rng(11)
    nodes = rng.integers(lo, hi - 1, size=(300, 3)).astype(np.int32)
    vel = rng.normal(0, 1, size=(300, 3)).astype(np.float32)
    for typ in (0, 1, 2):
        p = _params(np.eye(3), (0, 0, 0), (0, 0, 0), (0, 0, 0), 0.0, 1.0, friction, typ)
        vr, vo = _run_both(L, cfg, sdf, grad, p, np.float32(0.0), nodes, vel)
        if typ == 0:
            assert np.array_equal(vr.view(np.uint32), vo.view(np.uint32)) and (vo == 0).all()
        elif typ == 1:
            assert np.isnan(vr).all()
            assert np.array_equal(vo, vel)
        else:
            assert np.isfinite(vo).all() and (vo == 0).all()


def test_omega_changes_exactly_the_cross_product():
    """With omega = (0, 0, w) the reference's vec3_cross_vec3 gives (w r_y, w r_x, 0) where omega x r is (-w r_y, w r_x, 0):
    on a STICKY hit (velocity = object velocity) y and z are bit-identical and x differs by -2 w r_y, up to the rounding of
    the sum it enters; everything else is identical."""
    L = _ref()
    cfg = _cfg(L)
    sdf, grad = _field(cfg, "sphere")
    w = np.float32(1.7)
    t = np.float32(0.37)
    trans, trans_vel = np.float32([0.02, -0.01, 0.03]), np.float32([0.1, 0.2, -0.1])
    p = _params(np.eye(3), trans, trans_vel, (0, 0, w), 0.0, 1.0, 0.3, 0)
    nodes, vel = _queries(cfg, np.random.default_rng(5), n=3000)
    vr, vo = _run_both(L, cfg, sdf, grad, p, t, nodes, vel)
    hit = (vr != vel).any(1)
    assert hit.sum() > 50
    assert np.array_equal(vr[~hit], vo[~hit])
    assert np.array_equal(vr[:, 1:].view(np.uint32), vo[:, 1:].view(np.uint32))
    dx = np.float32(1.0 / (1 << cfg.domain_bits))
    b = trans + trans_vel * t
    ry = nodes[hit, 1].astype(np.float32) * dx - b[1]
    expect = np.float32(-2) * (w * ry)
    diff = vo[hit, 0].astype(np.float64) - vr[hit, 0].astype(np.float64)
    ulp = np.spacing(np.maximum(np.abs(vo[hit, 0]), np.abs(vr[hit, 0])).astype(np.float32)).astype(np.float64)
    assert np.all(np.abs(diff - expect) <= 4 * ulp + 1e-7)
    assert np.abs(expect).max() > 0.05


# ---- oracle physics -----------------------------------------------------------------------------------------------------------
def _cube_sim(cfg, lo, hi, v0, dt=5e-4):
    from claymore_b200 import samplers
    dx = 1.0 / (1 << cfg.domain_bits)
    pos = samplers.uniform_box(dx, np.round(np.asarray(lo) / dx).astype(int), np.round(np.asarray(hi) / dx).astype(int))
    s = cob.ColliderOracleSim(cfg, dt_default=dt, max_blocks=4000, threads=4)
    s.init_model(ob.FIXED_COROTATED, pos, np.float32(v0))
    return s, pos


def _field_collider(cfg, sdf, grad, typ, friction):
    col = cob.Collider()
    col.rot_mat[:] = [1, 0, 0, 0, 1, 0, 0, 0, 1]
    col.scale, col.type, col.friction = 1.0, typ, friction
    return col


def test_cube_dropped_on_sticky_box_stays_on_top():
    cfg = ob.make_config(domain_bits=6)
    ecfg = EngineConfig(domain_bits=6)
    top = 0.34
    sdf, grad = levelset.box(ecfg, (0.1, 0.1, 0.1), (0.9, top, 0.9))
    s, _ = _cube_sim(cfg, (0.42, 0.40, 0.42), (0.58, 0.52, 0.58), (0.0, -2.0, 0.0))
    s.set_collider(_field_collider(cfg, sdf, grad, 0, 0.3), sdf, grad)
    s.initial_setup()
    dx = 1.0 / 64
    lowest = 1.0
    for _ in range(20):
        s.step(10)
        lowest = min(lowest, s.retrieve(0)[:, 1].min())
    assert lowest >= top - dx, f"a particle went {top - lowest:.4f} below the collider's surface"
    assert lowest < top + 2 * dx, "the cube must reach the collider"
    assert s.sim_time == pytest.approx(200 * 5e-4, rel=1e-6)
    s.close()


def test_slip_half_space_keeps_tangential_velocity_without_friction():
    cfg = ob.make_config(domain_bits=6)
    ecfg = EngineConfig(domain_bits=6)
    floor = 0.36
    sdf, grad = levelset.plane(ecfg, (0.5, floor, 0.5), (0, 1, 0))
    results = {}
    for friction in (0.0, 0.3):
        s, pos = _cube_sim(cfg, (0.30, 0.37, 0.42), (0.42, 0.45, 0.54), (1.0, -1.0, 0.0))
        s.set_collider(_field_collider(cfg, sdf, grad, 1, friction), sdf, grad)
        s.initial_setup()
        x0 = s.retrieve(0)[:, 0].mean()
        s.step(160)
        results[friction] = (s.retrieve(0)[:, 0].mean() - x0) / s.sim_time
        s.close()
    assert results[0.0] == pytest.approx(1.0, abs=0.02), results
    assert results[0.3] < results[0.0] - 0.05, results


# ---- C ABI / adapter surface ----------------------------------------------------------------------------------------------------
def test_collider_symbols_exported_and_bound():
    import claymore_b200 as cb
    from claymore_b200 import _capi
    cb.build_library()
    lib = C.CDLL(cb.lib_path())
    for n in ("cb200_update_grid_velocity_query_max_collider", "cb200_sim_set_collider", "cb200_sim_clear_collider", "cb200_sim_time"):
        assert hasattr(lib, n), n
        assert n in _capi._SIGNATURES, n
    hdr = open(os.path.join(ROOT, "include", "claymore_b200.h")).read()
    body = re.search(r"typedef struct cb200_collider \{(.*?)\} cb200_collider;", hdr, re.S).group(1)
    assert C.sizeof(_capi.Collider) == C.sizeof(cob.Collider) == 8 + 4 * (9 + 3 + 3 + 3 + 3 + 1)
    assert "rot_mat[9]" in body
    assert re.search(r"CB200_STICKY = 0, CB200_SLIP = 1, CB200_SEPARATE = 2", hdr)


def test_adapter_collider_overload_compiles_against_boundary_condition(tmp_path):
    """The MGSP-form overload of update_grid_velocity_query_max takes the reference's SignedDistanceGrid as its Boundary."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.isdir(REFERENCE) or not os.path.exists(nvcc):
        pytest.skip("reference checkout or nvcc not available")
    tu = tmp_path / "adapter_collider_tu.cu"
    tu.write_text((r"""
#include <MnBase/Math/Matrix/Givens.cuh>
namespace mn { namespace math { template<typename T> __host__ __device__ void polar_decomposition(const std::array<T, 4>& a, GivensRotation<T>& r, std::array<T, 4>& s); }}
#include <claymore_b200_adapter.cuh>
// the reference's build defines these (asset directory; its fopen_s shim lives outside the collider's includes)
#define AssetDirPath ""
static inline int fopen_s(FILE** f, const char* n, const char* m) { *f = fopen(n, m); return *f ? 0 : 1; }
#include "BOUNDARY_CONDITION"
using namespace mn;
struct Ctx { cudaStream_t stream_compute() { return nullptr; } };
void collider_call(Ctx& cu, Partition<1>& part, GridBuffer& g0, SignedDistanceGrid& sdg, float* mv) {
    b200::compute_launch(cu, {8, 128}, b200::update_grid_velocity_query_max, (uint32_t) 8, g0, part, Duration(1e-4f), sdg, mv);
    b200::compute_launch(cu, {8, 128}, b200::update_grid_velocity_query_max, (uint32_t) 8, g0, part, Duration(1e-4f), mv);
}
""").replace("BOUNDARY_CONDITION", f"{REFERENCE}/Projects/MGSP/boundary_condition.cuh"))
    ref = REFERENCE
    fmt = tmp_path / "fmt"
    fmt.mkdir()
    (fmt / "core.h").write_text("#pragma once\nnamespace fmt { template<typename... A> inline void print(A&&...) {} }\n")
    (fmt / "color.h").write_text('#pragma once\n#include "core.h"\n')
    inc = [f"-I{tmp_path}", f"-I{ref}/Library", f"-I{ref}/Projects/GMPM", f"-I{ref}/Externals/function_ref", f"-I{ref}/Externals/optional", f"-I{ref}/Externals/variant", f"-I{ROOT}/include"]
    cmd = [nvcc, "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-extended-lambda", "--expt-relaxed-constexpr", "-DQR_CUH", "-include", "chrono",
           *inc, "-c", "-o", str(tmp_path / "adapter_collider_tu.o"), str(tu)]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-6000:]
