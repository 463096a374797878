"""ctypes binding of the CPU oracle with the boundaries: the signed-distance collider and the analytic collision objects
(oracle/libclaymore_collider_oracle.so).

TEST INFRASTRUCTURE ONLY.  The library holds the whole oracle plus the boundaries (oracle/collider_oracle.c), so a ColliderOracleSim
is an OracleSim whose calls go to that library; the plain oracle (oracle_binding) is left as it is.
"""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle_binding as ob
from claymore_b200._capi import CollisionObject

_ORACLE_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle")
_LIB_PATH = os.path.join(_ORACLE_DIR, "libclaymore_collider_oracle.so")
_SOURCES = ("collider_oracle.c", "collider_oracle.h", "claymore_oracle.c", "claymore_oracle.h")

STICKY, SLIP, SEPARATE = 0, 1, 2


class Collider(C.Structure):
    """orc_collider (layout of cb200_collider)."""
    _fields_ = [("sdf", C.c_void_p), ("rot_mat", C.c_float * 9), ("trans", C.c_float * 3), ("trans_vel", C.c_float * 3), ("omega", C.c_float * 3),
                ("dsdt", C.c_float), ("scale", C.c_float), ("friction", C.c_float), ("type", C.c_int)]


def build(force=False):
    newest = max(os.path.getmtime(os.path.join(_ORACLE_DIR, f)) for f in _SOURCES)
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < newest:
        subprocess.check_call(["make", "-C", _ORACLE_DIR, "-f", "collider.mk", "-s"])
    return _LIB_PATH


# the oracle entry points OracleSim and the kernel-level tests call, with the signatures oracle_binding gives them
_PLAIN = ["orc_sim_create", "orc_sim_destroy", "orc_sim_init_model", "orc_sim_initial_setup", "orc_sim_step", "orc_sim_counts", "orc_sim_dt",
          "orc_sim_max_vel", "orc_sim_retrieve", "orc_sim_active_keys", "orc_sim_grid", "orc_sim_particle_state", "orc_sim_update_fr_parameters",
          "orc_sim_update_sand_parameters", "orc_sim_update_j_fluid_parameters", "orc_sim_update_nacc_parameters", "orc_set_num_threads",
          "orc_sim_get_buffer", "orc_sim_get_partition", "orc_sim_get_grid", "orc_sim_bin_capacity", "orc_update_grid_velocity_query_max"]

_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        plain = ob.lib()
        for name in _PLAIN:
            src, dst = getattr(plain, name), getattr(L, name)
            dst.argtypes, dst.restype = src.argtypes, src.restype
        L.orc_collider_resolve.argtypes = [C.POINTER(ob.Config), C.POINTER(Collider), C.c_float, C.c_void_p, C.c_void_p]
        L.orc_update_grid_velocity_query_max_collider.argtypes = [C.POINTER(ob.Config), C.c_int, C.c_void_p, ob.Partition, C.c_float, C.POINTER(Collider), C.c_float, C.c_void_p]
        L.orc_update_grid_velocity_query_max_boundaries.argtypes = [C.POINTER(ob.Config), C.c_int, C.c_void_p, ob.Partition, C.c_float, C.POINTER(Collider),
                                                                    C.POINTER(CollisionObject), C.c_int, C.c_float, C.c_void_p]
        L.orc_csim_create.restype = C.c_void_p
        L.orc_csim_create.argtypes = [C.POINTER(ob.Config), C.c_float, C.c_int]
        L.orc_csim_destroy.argtypes = [C.c_void_p]
        L.orc_csim_sim.restype = C.c_void_p
        L.orc_csim_sim.argtypes = [C.c_void_p]
        L.orc_csim_set_collider.argtypes = [C.c_void_p, C.POINTER(Collider), C.c_void_p]
        L.orc_csim_clear_collider.argtypes = [C.c_void_p]
        L.orc_csim_set_objects.argtypes = [C.c_void_p, C.POINTER(CollisionObject), C.c_int]
        L.orc_csim_step.argtypes = [C.c_void_p, C.c_float]
        L.orc_csim_time.restype = C.c_double
        L.orc_csim_time.argtypes = [C.c_void_p]
        _lib = L
    return _lib


def unit_planes(objs):
    """copies of the objects (orc_collision_object: layout of cb200_collision_object) with plane normals made unit length in double, as
    cb200_sim_set_collision_objects stores them"""
    out = (CollisionObject * max(len(objs), 1))(*objs)
    for o in out[: len(objs)]:
        if o.shape == 0:
            n = np.asarray(list(o.b), np.float64)
            o.b[:] = [float(v) for v in n / np.sqrt((n * n).sum())]
    return out


class ColliderOracleSim(ob.OracleSim):
    """OracleSim with boundaries (a collider, then analytic collision objects); every call goes to the collider oracle's library."""

    def __init__(self, cfg, dt_default=1e-4, max_blocks=20000, threads=1):
        self.cfg = cfg
        self.max_blocks = max_blocks
        self.L = lib()
        self.L.orc_set_num_threads(threads)
        self.c = self.L.orc_csim_create(C.byref(cfg), dt_default, max_blocks)
        self.h = self.L.orc_csim_sim(self.c)
        self.materials = []
        self.counts = []

    def close(self):
        if self.c:
            self.L.orc_csim_destroy(self.c)
            self.c = self.h = None

    def step(self, n=1, time_left=1e30):
        for _ in range(n):
            self.L.orc_csim_step(self.c, time_left)

    def set_collider(self, col, sdf=None, grad=None):
        """col: Collider (its sdf field is ignored); sdf (N,N,N) + grad (3,N,N,N) on the 4G node lattice, or None to keep the field."""
        host = None
        if sdf is not None:
            host = np.ascontiguousarray(np.concatenate([np.asarray(sdf, np.float32).reshape(1, -1), np.asarray(grad, np.float32).reshape(3, -1)]))
        self.L.orc_csim_set_collider(self.c, C.byref(col), ob.ptr(host) if host is not None else None)

    def clear_collider(self):
        self.L.orc_csim_clear_collider(self.c)

    def set_collision_objects(self, objs):
        """objs: cb200_collision_object structs, resolved after the collider in list order; [] clears them"""
        self.L.orc_csim_set_objects(self.c, unit_planes(list(objs)), len(objs))

    @property
    def sim_time(self):
        return self.L.orc_csim_time(self.c)

