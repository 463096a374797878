"""GmpmSimulator-shaped host wrapper over the compiled step driver.

Mirrors the public interface of the reference's GmpmSimulator (Projects/GMPM/gmpm_simulator.cuh:121,168-254,303):
    GmpmSimulator(gpu, dt, fps, frames) ; init_model(material, positions, v0) ; update_*_parameters ; main_loop().
All compute happens in libclaymore_b200.so; this class only marshals arguments.
"""
import ctypes as C
import errno
import os

import numpy as np

from . import _capi
from ._capi import (CHANNELS, ERROR_OUTPUT_IO, OUTPUT_J, OUTPUT_V, SEPARATE, SLIP, STICKY, CollisionObject, Collider, Config, SimDesc,
                    SimStats, check, lib)

BOUNDARY_TYPES = {"sticky": STICKY, "slip": SLIP, "separate": SEPARATE}
OUTPUT_ATTRIBUTES = {"v": OUTPUT_V, "J": OUTPUT_J}


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
        self.restored = False
        self.emitters = []   # fn(sim, frame): called by main_loop at the start of each frame, before its sub-steps
        self._output_paths = []   # files of the frame being written (for the error of wait_output)
        self._levelsets = []      # the sdf.LevelSet of each registered lattice, in registry order

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

    def init_model_sdf(self, material, ls, offset, span, v0=(0.0, 0.0, 0.0), ppc=8, mode="random", seed=0):
        """init_model from a level set (claymore_b200.sdf.LevelSet): the particles are counted, the model allocated and the positions
        written on the device, with no host copy of them.  The node box must lie inside the domain (ValueError otherwise)."""
        from . import sdf
        sdf.check_box(ls, offset, span)
        smp = sdf.sampling(offset, span, ppc, mode, seed)
        phi = np.ascontiguousarray(ls.phi, dtype=np.float32)
        v = np.ascontiguousarray(v0, dtype=np.float32)
        mid, n = C.c_int(-1), C.c_int(0)
        check(self.L.cb200_sim_init_model_sdf(self.h, material, C.byref(ls.header), phi.ctypes.data_as(C.c_void_p), C.byref(smp),
                                              v.ctypes.data_as(C.c_void_p), C.byref(mid), C.byref(n)), "init_model_sdf")
        self.materials.append(material)
        self.counts.append(n.value)
        return mid.value

    # ---- sources: particles added to a set-up simulator at the current sub-step boundary (synchronises) -------------------
    EMIT_FILL = {"all": 0, "empty": _capi.EMIT_EMPTY_CELLS}

    def _fill(self, fill):
        if fill not in self.EMIT_FILL:
            raise ValueError(f"unknown fill {fill!r} (known: {', '.join(self.EMIT_FILL)})")
        return self.EMIT_FILL[fill]

    @staticmethod
    def _v0(v0):
        v = np.ascontiguousarray(v0, dtype=np.float32)
        if v.shape != (3,):
            raise ValueError(f"v0 must have 3 components, not shape {v.shape}")
        return v

    def add_particles(self, model, positions, v0=(0.0, 0.0, 0.0), fill="all"):
        """Appends particles to `model`, all with velocity v0 (the model starts them from F = I, as init_model).  fill="empty" keeps
        only positions whose cell held no particle of any model before the call.  Returns the count added.  The clock is kept;
        dt becomes min(dt, dx cfl / |v0|).  counts[model] grows by the count added; every model's library-side count becomes its
        live count, so counts stays an upper bound for sizing buffers, as it is once particles are lost."""
        flags = self._fill(fill)
        pos = np.ascontiguousarray(positions, dtype=np.float32).reshape(-1, 3)
        v = self._v0(v0)
        n = C.c_int(0)
        check(self.L.cb200_sim_add_particles(self.h, model, pos.ctypes.data_as(C.c_void_p), len(pos), v.ctypes.data_as(C.c_void_p), flags, C.byref(n)),
              "add_particles")
        self.counts[model] += n.value
        return n.value

    def add_particles_sdf(self, model, ls, offset, span, v0=(0.0, 0.0, 0.0), ppc=8, mode="random", seed=0, fill="all"):
        """add_particles with the positions sampled on the device from a level set, as init_model_sdf samples them."""
        from . import sdf
        flags = self._fill(fill)
        v = self._v0(v0)
        sdf.check_box(ls, offset, span)
        smp = sdf.sampling(offset, span, ppc, mode, seed)
        phi = np.ascontiguousarray(ls.phi, dtype=np.float32)
        n = C.c_int(0)
        check(self.L.cb200_sim_add_particles_sdf(self.h, model, C.byref(ls.header), phi.ctypes.data_as(C.c_void_p), C.byref(smp),
                                                 v.ctypes.data_as(C.c_void_p), flags, C.byref(n)), "add_particles_sdf")
        self.counts[model] += n.value
        return n.value

    # ---- sinks: particles removed from a set-up simulator at the current sub-step boundary (synchronises) -----------------
    def remove_particles(self, regions, models=None, outside=False):
        """Removes, from the models `models` (indices; default all of them), the particles whose position lies in any of `regions`
        (claymore_b200.objects constructors, placed at the simulated time; type and friction are ignored), or with outside=True the
        particles in none of them.  Survivors keep every channel and their velocity; the clock is kept.  Returns the count removed
        per model; counts drops by it.  An empty region list removes nothing."""
        from . import objects
        regions = list(regions)
        models = range(len(self.materials)) if models is None else list(models)
        mask = 0
        for m in models:
            if isinstance(m, bool) or not isinstance(m, (int, np.integer)) or not 0 <= m < len(self.materials):
                raise ValueError(f"unknown model {m!r} (the simulator has {len(self.materials)})")
            mask |= 1 << int(m)
        removed = (C.c_longlong * 8)()
        check(self.L.cb200_sim_remove_particles(self.h, mask, self._objects_array(regions), len(regions), _capi.REMOVE_OUTSIDE if outside else 0,
                                                removed), "remove_particles")
        return self._removed(removed)

    def remove_rows(self, model, mask):
        """Removes the rows of `model` where `mask` is true (non-zero); row i is row i of particle_state / retrieve now, and the mask
        has one entry per row.  Returns the count removed per model, as remove_particles."""
        m = np.ascontiguousarray(np.asarray(mask).reshape(-1) != 0, dtype=np.uint8)
        removed = (C.c_longlong * 8)()
        check(self.L.cb200_sim_remove_rows(self.h, model, m.ctypes.data_as(C.c_void_p), m.size, removed), "remove_rows")
        return self._removed(removed)

    def _removed(self, removed):
        out = [int(removed[m]) for m in range(len(self.materials))]
        for m, n in enumerate(out):
            self.counts[m] -= n
        return out

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

    def main_loop(self, on_frame=None, output=None, attributes=()):
        """initial_setup + nframes frames (gmpm_simulator.cuh:303-591).  output: a directory that receives every finished frame
        1..nframes as the reference's files (write_frame, `attributes` as there), written while the next frame runs; the loop waits
        for the last files before it returns.  on_frame(sim, frame) is called after each frame; every emitter (sim, frame) at the
        start of the frame, before its sub-steps (after the previous frame's files were queued).
        A restored simulator is set up already and runs only the frames after the ones its checkpoint had finished."""
        if not self.restored:
            self.initial_setup()
        for f in range(self.cur_frame + 1, self.nframes + 1):
            for emit in self.emitters:
                emit(self, f)
            self.advance_frame()
            if self.stats().error:
                break
            if output is not None:
                self.write_frame(output, f, attributes)
            if on_frame is not None:
                on_frame(self, f)
        if output is not None:
            self.wait_output()

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

    # ---- analytic collision objects (claymore_b200.objects, DESIGN.md section 2.9) ---------------------------------------------
    def set_collision_objects(self, objs):
        """Replaces the analytic collision objects by `objs` (claymore_b200.objects.plane / box / sphere / cylinder; [] clears them).
        From the next sub-step on the grid update resolves the level-set collider, then these in list order (synchronises)."""
        objs = list(objs)
        check(self.L.cb200_sim_set_collision_objects(self.h, self._objects_array(objs), len(objs)), "set_collision_objects")
        for i, o in enumerate(objs):
            tr = getattr(o, "track", None)
            if tr is not None:
                self.set_object_track(i, tr)

    def set_object_track(self, index, track):
        """Moves collision object `index` of the list set_collision_objects set along `track` (claymore_b200.objects.track; None
        clears it).  Resets the force report and synchronises (DESIGN.md section 2.14)."""
        if track is None:
            check(self.L.cb200_sim_set_object_track(self.h, int(index), None, 0, 0), "set_object_track")
        else:
            check(self.L.cb200_sim_set_object_track(self.h, int(index), track.keys, track.n, track.flags), "set_object_track")

    def clear_collision_objects(self):
        check(self.L.cb200_sim_set_collision_objects(self.h, None, 0), "clear_collision_objects")

    # ---- level-set collision objects (claymore_b200.objects.levelset, DESIGN.md section 2.11) -------------------------------
    def _objects_array(self, objs):
        """objects.array of `objs`, each objects.levelset entry with its level set's registry index: every level set not yet
        registered is registered once (its lattice stays on the device until clear_collision_levelsets or close).  Every object is
        validated before the first registration."""
        from . import objects
        objs = list(objs)
        objects.array(objs)
        out = []
        for o in objs:
            ls = getattr(o, "levelset", None)
            if ls is not None:
                o = CollisionObject.from_buffer_copy(o)
                o.b[1] = float(self.add_collision_levelset(ls))
            out.append(o)
        return objects.array(out, len(self._levelsets))

    def add_collision_levelset(self, ls):
        """Registry index of the level set `ls` (claymore_b200.sdf.LevelSet), registering it on first use (synchronises)."""
        for i, r in enumerate(self._levelsets):
            if r is ls:
                return i
        phi = np.ascontiguousarray(ls.phi, dtype=np.float32)
        idx = C.c_int(-1)
        check(self.L.cb200_sim_add_collision_levelset(self.h, C.byref(ls.header), phi.ctypes.data_as(C.c_void_p), C.byref(idx)),
              "add_collision_levelset")
        self._levelsets.append(ls)
        return idx.value

    def clear_collision_levelsets(self):
        """Frees every registered level set; refused (CB200Error) while a set collision object is a level set."""
        check(self.L.cb200_sim_clear_collision_levelsets(self.h), "clear_collision_levelsets")
        self._levelsets = []

    def sim_time(self):
        """Simulated time since initial_setup (sum of the dt of every finished sub-step)."""
        t = C.c_double(0.0)
        check(self.L.cb200_sim_time(self.h, C.byref(t)), "sim_time")
        return t.value

    # ---- boundary impulse report (DESIGN.md section 2.13) ---------------------------------------------------------------
    def report_forces(self, enable=True):
        """Turns the per-body impulse report of the grid update on or off and resets it (synchronises).  Body 0 is the level-set
        collider, body 1 + i collision object i."""
        check(self.L.cb200_sim_set_force_report(self.h, 1 if enable else 0), "report_forces")

    def collision_forces(self):
        """(elapsed, impulses) since the last reset, then resets: the simulated time covered and a float64 (1 + n_objects, 6) array
        of (Jx, Jy, Jz, Lx, Ly, Lz) per body, the impulse the material gave it and the angular impulse about its pivot
        trans + trans_vel t.  Mean force is J / elapsed, mean torque L / elapsed.  Synchronises; needs report_forces()."""
        out = np.zeros((_capi.MAX_COLLISION_OBJECTS + 1, _capi.FORCE_COMPONENTS), np.float64)
        n, elapsed = C.c_int(0), C.c_double(0.0)
        check(self.L.cb200_sim_collision_forces(self.h, out.ctypes.data_as(C.c_void_p), len(out), C.byref(n), C.byref(elapsed)), "collision_forces")
        return elapsed.value, out[:n.value].copy()

    # ---- checkpoint / restore (format: include/claymore_b200.h, reader: claymore_b200.checkpoint) -------------------
    def checkpoint_begin(self):
        """Snapshot at the current sub-step boundary; returns the blob's size without waiting for its copy to the host, so
        sub-steps issued before checkpoint_end overlap with it."""
        n = C.c_size_t(0)
        check(self.L.cb200_sim_checkpoint_begin(self.h, C.byref(n)), "checkpoint_begin")
        return n.value

    def checkpoint_end(self, path=None):
        """Waits for the copy of the last checkpoint_begin.  Writes the blob to `path`, or returns a copy of it (uint8 array)."""
        p, n = C.c_void_p(), C.c_size_t(0)
        check(self.L.cb200_sim_checkpoint_end(self.h, C.byref(p), C.byref(n)), "checkpoint_end")
        blob = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_ubyte)), shape=(n.value,))
        if path is None:
            return blob.copy()
        with open(path, "wb") as f:
            f.write(memoryview(blob))
        return n.value

    def save_checkpoint(self, path=None):
        """checkpoint_begin + checkpoint_end: the whole state at this sub-step boundary to `path` (or returned as bytes)."""
        self.checkpoint_begin()
        return self.checkpoint_end(path)

    @classmethod
    def from_checkpoint(cls, path, **overrides):
        """A simulator matching a checkpoint (config, dt_default, fps, MGSP rank / world; capacity defaults to the saved one),
        not yet restored: set a collider or wire MGSP peers, then call restore(path)."""
        from . import checkpoint
        inf = checkpoint.inspect(path)[0]
        c = inf.cfg
        kw = dict(dt=inf.dt_default, fps=inf.fps, config=Config(c.domain_bits, c.max_ppc, c.boundary, c.gravity, c.cfl), max_blocks=inf.max_blocks,
                  mgsp_rank=inf.mgsp_rank, mgsp_world=inf.mgsp_world)
        kw.update(overrides)
        return cls(**kw)

    def restore(self, path_or_blob, setup=True):
        """In place of init_model + initial_setup: the models, grid and clock of a checkpoint (file path or blob).
        setup=False only registers the models and stages their state (in place of init_model); initial_setup() then restores.
        MGSP ranks sharing a device in one process do that on every rank first, then run initial_setup concurrently."""
        from . import checkpoint
        inf, blob = checkpoint.inspect(path_or_blob)
        data = np.ascontiguousarray(blob)   # one read of the file; the library copies it to the device
        fn = self.L.cb200_sim_restore if setup else self.L.cb200_sim_restore_models
        check(fn(self.h, data.ctypes.data_as(C.c_void_p), data.size), "restore")
        self.materials = [m.material for m in inf.models[: inf.n_models]]
        self.counts = [m.count for m in inf.models[: inf.n_models]]
        self.cur_frame = inf.frames
        self.restored = True

    # ---- per-frame .bgeo output (output_model + write_partio; reader: claymore_b200.bgeo) --------------------------------------
    def frame_paths(self, directory, frame):
        """The reference's file names, model_id[i]_frame[f].bgeo; an MGSP rank adds itself: model_id[i]_rank[r]_frame[f].bgeo."""
        rank = f"_rank[{self.mgsp_rank}]" if self.mgsp_world > 1 else ""
        return [os.path.join(directory, f"model_id[{i}]{rank}_frame[{frame}].bgeo") for i in range(len(self.materials))]

    def write_frame(self, directory, frame=None, attributes=()):
        """One .bgeo file per model of the particles at this sub-step boundary, in `directory` (frame defaults to the current
        frame).  attributes: any of "v" (velocity, VECTOR 3) and "J" (volume ratio, FLOAT 1).  Returns once the particles are
        gathered; the files are written by the simulator's writer thread while later sub-steps run.  One frame is in flight: a
        call while the previous frame is still being written waits for it.  Returns the paths."""
        bits = 0
        for a in attributes:
            if a not in OUTPUT_ATTRIBUTES:
                raise ValueError(f"unknown output attribute {a!r} (known: {', '.join(OUTPUT_ATTRIBUTES)})")
            bits |= OUTPUT_ATTRIBUTES[a]
        paths = self.frame_paths(directory, self.cur_frame if frame is None else frame)
        arr = (C.c_char_p * len(paths))(*[os.fsencode(p) for p in paths])
        err = self.L.cb200_sim_frame_output(self.h, arr, bits)
        if err == ERROR_OUTPUT_IO:   # an earlier frame failed: raise its error (nothing of this frame was queued)
            self.wait_output()
        check(err, "frame_output")
        self._output_paths = paths
        return paths

    def wait_output(self):
        """Waits until the files of the last write_frame are written.  Raises OSError (with the path) when one failed."""
        e = C.c_int(0)
        err = self.L.cb200_sim_frame_output_wait(self.h, C.byref(e))
        paths, self._output_paths = self._output_paths, []
        if err == ERROR_OUTPUT_IO:
            missing = [p for p in paths if not os.path.exists(p)]   # a file that failed is removed
            path = missing[0] if missing else (paths[0] if paths else None)
            raise OSError(e.value or errno.EIO, os.strerror(e.value or errno.EIO), path)
        check(err, "frame_output_wait")

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
        if n.value == 0:   # an emptied model: there may be no staging buffer to view
            return np.zeros((0, 3), np.float32)
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
