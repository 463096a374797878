"""GmpmSimulator-shaped host wrapper over the compiled step driver.

Mirrors the public interface of the reference's GmpmSimulator (Projects/GMPM/gmpm_simulator.cuh:121,168-254,303):
    GmpmSimulator(gpu, dt, fps, frames) ; init_model(material, positions, v0) ; update_*_parameters ; main_loop().
All compute happens in libclaymore_b200.so; this class only marshals arguments.
"""
import ctypes as C

import numpy as np

from . import _capi
from ._capi import CHANNELS, SEPARATE, SLIP, STICKY, Collider, Config, SimDesc, SimStats, check, lib

BOUNDARY_TYPES = {"sticky": STICKY, "slip": SLIP, "separate": SEPARATE}


class GmpmSimulator:
    DEFAULT_DT = 1e-4     # gmpm_simulator.cuh:24
    DEFAULT_FPS = 24      # :25
    DEFAULT_FRAMES = 60   # :26
    MGSP_HANDLE_BYTES = 160   # CB200_MGSP_HANDLE_BYTES

    def __init__(self, gpu=0, dt=DEFAULT_DT, fps=DEFAULT_FPS, frames=DEFAULT_FRAMES, config=None, max_blocks=10000, use_graph=True,
                 stream=None, mgsp_rank=0, mgsp_world=1, mgsp_halo_cap=0, auto_grow=None):
        self.L = lib()
        self.gpu = gpu
        self.cfg = config if config is not None else Config()
        self.fps, self.nframes = fps, frames
        if auto_grow is None:   # the reference checks its capacities every sub-step (gmpm_simulator.cuh:331); MGSP buffers are peer-mapped
            auto_grow = mgsp_world <= 1
        self.desc = SimDesc(self.cfg, dt, fps, max_blocks, 1 if use_graph else 0, mgsp_rank, mgsp_world, mgsp_halo_cap, 1 if auto_grow else 0)
        self.mgsp_rank, self.mgsp_world = mgsp_rank, mgsp_world
        self.max_blocks = max_blocks
        self._stream = C.c_void_p(stream) if stream else C.c_void_p(0)
        self.h = C.c_void_p()
        check(self.L.cb200_sim_create(C.byref(self.desc), self._stream, C.byref(self.h)), "cb200_sim_create")
        self.materials, self.counts = [], []
        self.cur_frame = 0

    # ---- lifecycle -------------------------------------------------------------------------------
    def close(self):
        if getattr(self, "h", None) and self.h.value:
            self.L.cb200_sim_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- model / material API (gmpm_simulator.cuh:168-254) ----------------------------------------
    def init_model(self, material, positions, v0=(0.0, 0.0, 0.0)):
        pos = np.ascontiguousarray(positions, dtype=np.float32).reshape(-1, 3)
        v = np.ascontiguousarray(v0, dtype=np.float32)
        mid = C.c_int(-1)
        check(self.L.cb200_sim_init_model(self.h, material, pos.ctypes.data_as(C.c_void_p), len(pos), v.ctypes.data_as(C.c_void_p), C.byref(mid)), "init_model")
        self.materials.append(material)
        self.counts.append(len(pos))
        return mid.value

    def update_fr_parameters(self, rho, vol, ym, pr, model=-1):
        check(self.L.cb200_sim_update_fr_parameters(self.h, self._m(model), rho, vol, ym, pr), "update_fr_parameters")

    def update_sand_parameters(self, rho, vol, ym, pr, model=-1):
        check(self.L.cb200_sim_update_sand_parameters(self.h, self._m(model), rho, vol, ym, pr), "update_sand_parameters")

    def update_j_fluid_parameters(self, rho, vol, bulk, gamma, visc, model=-1):
        check(self.L.cb200_sim_update_j_fluid_parameters(self.h, self._m(model), rho, vol, bulk, gamma, visc), "update_j_fluid_parameters")

    def update_nacc_parameters(self, rho, vol, ym, pr, beta, xi, model=-1):
        check(self.L.cb200_sim_update_nacc_parameters(self.h, self._m(model), rho, vol, ym, pr, beta, xi), "update_nacc_parameters")

    def _m(self, model):
        return len(self.materials) - 1 if model < 0 else model

    # ---- stepping -----------------------------------------------------------------------------------
    def initial_setup(self):
        check(self.L.cb200_sim_initial_setup(self.h), "initial_setup")

    def step(self, n=1):
        """n sub-steps (asynchronous)."""
        check(self.L.cb200_sim_step(self.h, n), "step")

    def advance_frame(self):
        n = C.c_int(0)
        check(self.L.cb200_sim_advance_frame(self.h, C.byref(n)), "advance_frame")
        self.cur_frame += 1
        return n.value

    def main_loop(self, on_frame=None):
        """initial_setup + nframes frames (gmpm_simulator.cuh:303-591); on_frame(sim, frame) replaces the bgeo dump."""
        self.initial_setup()
        for f in range(1, self.nframes + 1):
            self.advance_frame()
            if self.stats().error:
                break
            if on_frame is not None:
                on_frame(self, f)

    def sync(self):
        check(self.L.cb200_sim_sync(self.h), "sync")

    # ---- capacity (check_capacity + resizes, gmpm_simulator.cuh:283-300) -----------------------------
    def reserve(self, max_blocks):
        check(self.L.cb200_sim_reserve(self.h, int(max_blocks)), "reserve")
        self.max_blocks = self.capacity()[0]

    def check_capacity(self):
        """Applies the reference's rule (exterior blocks > 3/4 capacity -> capacity x 3/2); returns the new capacity or 0."""
        g = C.c_int(0)
        check(self.L.cb200_sim_check_capacity(self.h, C.byref(g)), "check_capacity")
        if g.value:
            self.max_blocks = g.value
        return g.value

    def capacity(self):
        mb, ev = C.c_int(0), C.c_int(0)
        check(self.L.cb200_sim_capacity(self.h, C.byref(mb), C.byref(ev)), "capacity")
        return mb.value, ev.value

    # ---- signed-distance collider (SignedDistanceGrid, Projects/MGSP/boundary_condition.cuh:25-250) -------------------
    def set_collider(self, sdf=None, grad=None, type="sticky", friction=0.3, trans=(0.0, 0.0, 0.0), trans_vel=(0.0, 0.0, 0.0),
                     omega=(0.0, 0.0, 0.0), rot=None, scale=1.0, dsdt=0.0):
        """One collision object acting on the grid update from the next sub-step on (synchronises).  sdf: (N, N, N) signed
        distance on the N = 4G grid nodes, grad: (3, N, N, N) its gradient (see levelset); both None keep the field set before.
        type: "sticky" / "slip" / "separate" or CB200_*; rot: 3x3 rotation (row i, column j = rot_mat(i, j)).  Defaults are
        SignedDistanceGrid's (:38-49).  The collider is placed at the simulated time at the start of each sub-step."""
        col = Collider()
        col.type = BOUNDARY_TYPES[type] if isinstance(type, str) else int(type)
        col.rot_mat[:] = [float(v) for v in np.asarray(np.eye(3) if rot is None else rot, dtype=np.float64).reshape(9)]
        col.trans[:], col.trans_vel[:], col.omega[:] = [float(v) for v in trans], [float(v) for v in trans_vel], [float(v) for v in omega]
        col.dsdt, col.scale, col.friction = dsdt, scale, friction
        host = None
        if sdf is not None:
            n = 4 * self.cfg.grid_size
            host = np.ascontiguousarray(np.concatenate([np.asarray(sdf, np.float32).reshape(1, -1), np.asarray(grad, np.float32).reshape(3, -1)]))
            if host.shape != (4, n ** 3):
                raise ValueError(f"level set must be {n}^3 nodes (distance) and 3 x {n}^3 (gradient)")
        check(self.L.cb200_sim_set_collider(self.h, C.byref(col), host.ctypes.data_as(C.c_void_p) if host is not None else None), "set_collider")

    def clear_collider(self):
        check(self.L.cb200_sim_clear_collider(self.h), "clear_collider")

    def sim_time(self):
        """Simulated time since initial_setup (sum of the dt of every finished sub-step)."""
        t = C.c_double(0.0)
        check(self.L.cb200_sim_time(self.h, C.byref(t)), "sim_time")
        return t.value

    # ---- observation --------------------------------------------------------------------------------
    def stats(self):
        st = SimStats()
        check(self.L.cb200_sim_stats_get(self.h, C.byref(st)), "stats")
        return st

    def block_counts(self):
        st = self.stats()
        return st.particle_block_count, st.neighbor_block_count, st.exterior_block_count

    def retrieve(self, model, copy=True, out=None):
        """Positions of one model (output_model).  out: caller-owned float32 array of shape (count, 3) (pinned memory makes
        the device->host copy fast); otherwise copy=False returns a view of the simulator's pinned staging buffer, valid until
        the next retrieve of that model."""
        n, p = C.c_int(0), C.c_void_p()
        if out is not None:
            assert out.dtype == np.float32 and out.size >= 3 * self.counts[model] and out.flags.c_contiguous
            check(self.L.cb200_sim_retrieve(self.h, model, out.ctypes.data_as(C.c_void_p), C.byref(n)), "retrieve")
            return out.reshape(-1, 3)[: n.value]
        check(self.L.cb200_sim_retrieve_pinned(self.h, model, C.byref(p), C.byref(n)), "retrieve")
        view = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_float)), shape=(n.value, 3))
        return view.copy() if copy else view

    def particle_state(self, model):
        nch = CHANNELS[self.materials[model]]
        out = np.zeros((self.counts[model], nch), np.float32)
        n = C.c_int(0)
        check(self.L.cb200_sim_particle_state(self.h, model, out.ctypes.data_as(C.c_void_p), C.byref(n)), "particle_state")
        return out[: n.value]

    def active_keys(self):
        self.max_blocks = self.capacity()[0]
        out = np.zeros((self.max_blocks, 3), np.int32)
        n = C.c_int(0)
        check(self.L.cb200_sim_active_keys(self.h, out.ctypes.data_as(C.c_void_p), self.max_blocks, C.byref(n)), "active_keys")
        return out[: n.value]

    def grid(self):
        self.max_blocks = self.capacity()[0]
        out = np.zeros((self.max_blocks, 4, 64), np.float32)
        n = C.c_int(0)
        check(self.L.cb200_sim_grid(self.h, out.ctypes.data_as(C.c_void_p), self.max_blocks, C.byref(n)), "grid")
        return out[: n.value]

    # ---- MGSP peer wiring (one process per GPU: exchange the 64-byte IPC handles with any host all-gather) ----------
    def mgsp_ipc_handle(self):
        buf = (C.c_ubyte * self.MGSP_HANDLE_BYTES)()
        check(self.L.cb200_sim_mgsp_ipc_handle(self.h, buf), "mgsp_ipc_handle")
        return bytes(buf)

    def mgsp_open_peers(self, handles_by_rank):
        blob = b"".join(handles_by_rank)
        assert len(blob) == self.MGSP_HANDLE_BYTES * self.mgsp_world
        buf = (C.c_ubyte * len(blob)).from_buffer_copy(blob)
        check(self.L.cb200_sim_mgsp_open_peers(self.h, buf), "mgsp_open_peers")

    def mgsp_inbox(self):
        """(inbox pointer, next-grid pointer) of this rank, for peers living in the same process."""
        p, g, n = C.c_void_p(), C.c_void_p(), C.c_size_t()
        check(self.L.cb200_sim_mgsp_inbox(self.h, C.byref(p), C.byref(g), C.byref(n)), "mgsp_inbox")
        return p.value, g.value

    def mgsp_set_peers(self, ptrs_by_rank):
        a = (C.c_void_p * len(ptrs_by_rank))(*[p[0] for p in ptrs_by_rank])
        b = (C.c_void_p * len(ptrs_by_rank))(*[p[1] for p in ptrs_by_rank])
        check(self.L.cb200_sim_mgsp_set_peers(self.h, a, b), "mgsp_set_peers")

    def mgsp_halo_counts(self):
        cnt = (C.c_int * max(self.mgsp_world, 1))()
        hp = C.c_int(0)
        check(self.L.cb200_sim_mgsp_halo_counts(self.h, cnt, C.byref(hp)), "mgsp_halo_counts")
        return list(cnt), hp.value

    def profile(self, enable=True):
        """CUDA-event pairs around every g2p2g launch (sub-steps run as plain stream launches meanwhile)."""
        check(self.L.cb200_sim_profile(self.h, 1 if enable else 0), "profile")

    def profile_read(self):
        ms, n = C.c_double(0.0), C.c_int(0)
        check(self.L.cb200_sim_profile_read(self.h, C.byref(ms), C.byref(n)), "profile_read")
        return ms.value, n.value

    # phase id of cb200_sim_profile_phases -> name, in sub-step order; ids 6 and 8 are recorded by multi-GPU (MGSP) runs only
    PHASES = {1: "grid_update", 5: "g2p2g", 6: "halo_done_publish", 7: "rebuild", 9: "carry_exterior_finalize", 8: "halo_tagging"}
    MGSP_PHASES = (6, 8)

    def profile_phases(self):
        """{phase: summed ms} over the sub-steps issued while profile(True) was on (call before profile_read)."""
        out = (C.c_double * 10)()
        check(self.L.cb200_sim_profile_phases(self.h, out), "profile_phases")
        return {n: out[i] for i, n in self.PHASES.items() if self.mgsp_world > 1 or i not in self.MGSP_PHASES}

    @property
    def launch_count(self):
        return int(self.L.cb200_sim_launch_count(self.h))
