"""ctypes binding of the CPU oracle with the analytic collision objects (tests/oracle_objects/objects_oracle.c).

TEST INFRASTRUCTURE ONLY.  The library holds the whole collider oracle plus the objects; it is compiled on first use into a
temporary directory (keyed by the sources' contents), so that the checkout is never written to.  ObjectsOracleSim is a
ColliderOracleSim whose sub-step is the objects form."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import collider_oracle_binding as cob
import oracle_binding as ob
from claymore_b200._capi import CollisionObject

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE_DIR = os.path.join(os.path.dirname(_HERE), "oracle")
_SOURCE = os.path.join(_HERE, "oracle_objects", "objects_oracle.c")
_DEPS = [_SOURCE] + [os.path.join(_ORACLE_DIR, f) for f in ("collider_oracle.c", "collider_oracle.h", "claymore_oracle.c", "claymore_oracle.h")]
CFLAGS = ["-O2", "-std=c99", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math"]   # the oracle's own flags (oracle/collider.mk)

_lib = None


def build():
    h = hashlib.sha256()
    for f in _DEPS:
        h.update(open(f, "rb").read())
    out = os.path.join(tempfile.gettempdir(), f"cb200_objects_oracle_{h.hexdigest()[:16]}_{os.getuid()}.so")
    if not os.path.exists(out):
        tmp = out + f".{os.getpid()}.tmp"
        subprocess.check_call(["gcc", *CFLAGS, "-I", _ORACLE_DIR, "-shared", "-o", tmp, _SOURCE, "-lm"])
        os.replace(tmp, out)
    return out


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        plain = ob.lib()
        for name in cob._PLAIN:
            src, dst = getattr(plain, name), getattr(L, name)
            dst.argtypes, dst.restype = src.argtypes, src.restype
        P = C.POINTER(CollisionObject)
        L.orc_objects_resolve.argtypes = [C.POINTER(ob.Config), C.POINTER(cob.Collider), P, C.c_int, C.c_float, C.c_void_p, C.c_void_p]
        L.orc_update_grid_velocity_query_max_objects.argtypes = [C.POINTER(ob.Config), C.c_int, C.c_void_p, ob.Partition, C.c_float, C.POINTER(cob.Collider), P, C.c_int,
                                                                 C.c_float, C.c_void_p]
        L.orc_csim_create.restype = C.c_void_p
        L.orc_csim_create.argtypes = [C.POINTER(ob.Config), C.c_float, C.c_int]
        L.orc_csim_destroy.argtypes = [C.c_void_p]
        L.orc_csim_sim.restype = C.c_void_p
        L.orc_csim_sim.argtypes = [C.c_void_p]
        L.orc_csim_set_collider.argtypes = [C.c_void_p, C.POINTER(cob.Collider), C.c_void_p]
        L.orc_csim_clear_collider.argtypes = [C.c_void_p]
        L.orc_csim_step_objects.argtypes = [C.c_void_p, P, C.c_int, C.c_float]
        L.orc_csim_time.restype = C.c_double
        L.orc_csim_time.argtypes = [C.c_void_p]
        _lib = L
    return _lib


def unit_planes(objs):
    """copies of the objects with plane normals made unit length in double, as cb200_sim_set_collision_objects stores them"""
    import numpy as np
    out = (CollisionObject * max(len(objs), 1))(*objs)
    for o in out[: len(objs)]:
        if o.shape == 0:
            n = np.asarray(list(o.b), np.float64)
            o.b[:] = [float(v) for v in n / np.sqrt((n * n).sum())]
    return out


class ObjectsOracleSim(cob.ColliderOracleSim):
    """ColliderOracleSim with analytic collision objects after its collider."""

    def __init__(self, cfg, dt_default=1e-4, max_blocks=20000, threads=1):
        self.cfg = cfg
        self.max_blocks = max_blocks
        self.L = lib()
        self.L.orc_set_num_threads(threads)
        self.c = self.L.orc_csim_create(C.byref(cfg), dt_default, max_blocks)
        self.h = self.L.orc_csim_sim(self.c)
        self.materials = []
        self.counts = []
        self.set_collision_objects([])

    def set_collision_objects(self, objs):
        self._n = len(objs)
        self._objs = unit_planes(list(objs))

    def step(self, n=1, time_left=1e30):
        for _ in range(n):
            self.L.orc_csim_step_objects(self.c, self._objs, self._n, time_left)


def build_oracle(scene, dt=1e-4, max_blocks=4000, max_ppc=128, threads=1, cfl=0.5):
    """tests/scenes.build_oracle with an ObjectsOracleSim"""
    import scenes
    cfg = ob.make_config(domain_bits=scene["domain_bits"], max_ppc=max_ppc, cfl=cfl)
    sim = ObjectsOracleSim(cfg, dt, max_blocks, threads=threads)
    dx = 1.0 / (1 << scene["domain_bits"])
    for m in scene["models"]:
        mid = sim.init_model(m["material"], m["pos"], m["v0"])
        scenes.apply_material(sim, mid, m["material"], dx, True)
    sim.initial_setup()
    return sim
