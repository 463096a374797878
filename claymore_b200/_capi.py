"""ctypes binding of libclaymore_b200.so (C ABI declared in include/claymore_b200.h)."""
import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, "lib", "libclaymore_b200.so")

J_FLUID, FIXED_COROTATED, SAND, NACC = 0, 1, 2, 3
CHANNELS = {J_FLUID: 4, FIXED_COROTATED: 12, SAND: 13, NACC: 13}
BIN_FLOATS = {J_FLUID: 128, FIXED_COROTATED: 512, SAND: 512, NACC: 512}


class CB200Error(RuntimeError):
    pass


class Config(C.Structure):
    """cb200_config: runtime form of claymore's compile-time `namespace config` (Projects/GMPM/settings.h)."""
    _fields_ = [("domain_bits", C.c_int), ("max_ppc", C.c_int), ("boundary", C.c_int), ("gravity", C.c_float), ("cfl", C.c_float)]

    def __init__(self, domain_bits=8, max_ppc=128, boundary=2, gravity=-9.8, cfl=0.5):
        super().__init__(domain_bits, max_ppc, boundary, gravity, cfl)

    @property
    def dx(self):
        return 1.0 / (1 << self.domain_bits)

    @property
    def grid_size(self):
        return 1 << (self.domain_bits - 2)

    @property
    def ppb(self):
        return 64 * self.max_ppc


class ParticleBuffer(C.Structure):
    """cb200_particle_buffer: ParticleBuffer<M> by-value fields (Projects/GMPM/particle_buffer.cuh:38-264)."""
    _fields_ = [
        ("material", C.c_int),
        ("bins", C.c_void_p), ("cell_particle_counts", C.c_void_p), ("particle_bucket_sizes", C.c_void_p),
        ("cellbuckets", C.c_void_p), ("blockbuckets", C.c_void_p), ("bin_offsets", C.c_void_p),
        ("rho", C.c_float), ("volume", C.c_float), ("mass", C.c_float),
        ("bulk", C.c_float), ("gamma", C.c_float), ("viscosity", C.c_float),
        ("lambda_", C.c_float), ("mu", C.c_float),
        ("cohesion", C.c_float), ("beta", C.c_float), ("yield_surface", C.c_float), ("volume_correction", C.c_int),
        ("bm", C.c_float), ("xi", C.c_float), ("msqr", C.c_float), ("hardening_on", C.c_int),
    ]


class Partition(C.Structure):
    """cb200_partition: Partition<1> by-value fields (Projects/GMPM/hash_table.cuh:27-135)."""
    _fields_ = [("count", C.c_void_p), ("index_table", C.c_void_p), ("active_keys", C.c_void_p),
                ("halo_count", C.c_void_p), ("halo_marks", C.c_void_p), ("overlap_marks", C.c_void_p), ("halo_blocks", C.c_void_p)]


class SimDesc(C.Structure):
    _fields_ = [("cfg", Config), ("dt_default", C.c_float), ("fps", C.c_int), ("max_blocks", C.c_int), ("use_graph", C.c_int),
                ("mgsp_rank", C.c_int), ("mgsp_world", C.c_int), ("mgsp_halo_cap", C.c_int), ("auto_grow", C.c_int)]


class SimStats(C.Structure):
    _fields_ = [("particle_block_count", C.c_int), ("neighbor_block_count", C.c_int), ("exterior_block_count", C.c_int),
                ("bin_count", C.c_int * 8), ("dt", C.c_float), ("next_dt", C.c_float), ("max_vel", C.c_float), ("step_time", C.c_float),
                ("error", C.c_int), ("steps", C.c_longlong)]


STICKY, SLIP, SEPARATE = 0, 1, 2   # BoundaryT, Projects/MGSP/boundary_condition.cuh:18-22


class Collider(C.Structure):
    """cb200_collider: SignedDistanceGrid's members (Projects/MGSP/boundary_condition.cuh:28-35) + the device field pointer."""
    _fields_ = [("sdf", C.c_void_p), ("rot_mat", C.c_float * 9), ("trans", C.c_float * 3), ("trans_vel", C.c_float * 3), ("omega", C.c_float * 3),
                ("dsdt", C.c_float), ("scale", C.c_float), ("friction", C.c_float), ("type", C.c_int)]


def lib_path():
    return _LIB


def build_library(force=False):
    """Compile csrc/ for sm_90a with nvcc (in-tree, so the .so travels with the repo snapshot)."""
    src = os.path.join(_HERE, "csrc")
    if force:
        subprocess.check_call(["make", "-C", src, "-s", "clean"])
    subprocess.check_call(["make", "-C", src, "-s"])
    return _LIB


_lib = None

_P, _I, _F = C.c_void_p, C.c_int, C.c_float
_CFG = C.POINTER(Config)

_SIGNATURES = {
    "cb200_g2p2g": [_CFG, _F, _F, _I, ParticleBuffer, ParticleBuffer, Partition, Partition, _P, _P, _P],
    "cb200_update_grid_velocity_query_max": [_CFG, _I, _P, Partition, _F, _P, _P],
    "cb200_update_grid_velocity_query_max_collider": [_CFG, _I, _P, Partition, _F, C.POINTER(Collider), _F, _P, _P],
    "cb200_clear_grid": [_I, _P, _P],
    "cb200_cell_bucket_to_block": [_CFG, _I, _P, _P, _P, _P, _P],
    "cb200_mark_active_grid_blocks": [_I, _P, _P, _P],
    "cb200_mark_active_particle_blocks": [_I, _P, _P, _P],
    "cb200_exclusive_scan": [_I, _P, _P, _P],
    "cb200_exclusive_scan_inverse": [_I, _P, _P, _P],
    "cb200_update_partition": [_CFG, _I, _P, Partition, Partition, _P],
    "cb200_update_buckets": [_CFG, _I, _P, ParticleBuffer, ParticleBuffer, _P],
    "cb200_compute_bin_capacity": [_I, _P, _P, _P],
    "cb200_register_neighbor_blocks": [_CFG, _I, Partition, _P],
    "cb200_register_exterior_blocks": [_CFG, _I, Partition, _P],
    "cb200_copy_selected_grid_blocks": [_CFG, _I, _P, Partition, _P, _P, _P, _P],
    "cb200_reset_table": [_CFG, Partition, _P],
    "cb200_activate_blocks": [_CFG, _I, _P, Partition, _P],
    "cb200_build_particle_cell_buckets": [_CFG, _I, _P, ParticleBuffer, Partition, _P],
    "cb200_array_to_buffer": [_CFG, _I, _P, ParticleBuffer, _P],
    "cb200_rasterize": [_CFG, _I, _P, _P, Partition, _F, _P, _P],
    "cb200_init_adv_bucket": [_CFG, _I, _P, _P, _P],
    "cb200_retrieve_particle_buffer": [_CFG, _I, Partition, Partition, ParticleBuffer, ParticleBuffer, _P, _P, _P],
    "cb200_mark_overlapping_blocks": [_CFG, _I, _I, _P, Partition, _P, _P, _P],
    "cb200_collect_blockids_for_halo_reduction": [_CFG, _I, Partition, _P],
    "cb200_collect_grid_blocks": [_CFG, _I, _P, _P, Partition, _P, _P],
    "cb200_reduce_grid_blocks": [_CFG, _I, _P, _P, Partition, _P, _P],
    "cb200_sim_create": [C.POINTER(SimDesc), _P, C.POINTER(_P)],
    "cb200_sim_destroy": [_P],
    "cb200_sim_init_model": [_P, _I, _P, _I, _P, C.POINTER(_I)],
    "cb200_sim_update_fr_parameters": [_P, _I, _F, _F, _F, _F],
    "cb200_sim_update_sand_parameters": [_P, _I, _F, _F, _F, _F],
    "cb200_sim_update_j_fluid_parameters": [_P, _I, _F, _F, _F, _F, _F],
    "cb200_sim_update_nacc_parameters": [_P, _I, _F, _F, _F, _F, _F, _F],
    "cb200_sim_initial_setup": [_P],
    "cb200_sim_step": [_P, _I],
    "cb200_sim_advance_frame": [_P, C.POINTER(_I)],
    "cb200_sim_sync": [_P],
    "cb200_sim_reserve": [_P, _I],
    "cb200_sim_check_capacity": [_P, C.POINTER(_I)],
    "cb200_sim_capacity": [_P, C.POINTER(_I), C.POINTER(_I)],
    "cb200_sim_stats_get": [_P, C.POINTER(SimStats)],
    "cb200_sim_retrieve": [_P, _I, _P, C.POINTER(_I)],
    "cb200_sim_retrieve_pinned": [_P, _I, C.POINTER(_P), C.POINTER(_I)],
    "cb200_sim_particle_state": [_P, _I, _P, C.POINTER(_I)],
    "cb200_sim_active_keys": [_P, _P, _I, C.POINTER(_I)],
    "cb200_sim_grid": [_P, _P, _I, C.POINTER(_I)],
    "cb200_sim_set_collider": [_P, C.POINTER(Collider), _P],
    "cb200_sim_clear_collider": [_P],
    "cb200_sim_time": [_P, C.POINTER(C.c_double)],
    "cb200_sim_mgsp_inbox": [_P, C.POINTER(_P), C.POINTER(_P), C.POINTER(C.c_size_t)],
    "cb200_sim_mgsp_ipc_handle": [_P, _P],
    "cb200_sim_mgsp_open_peers": [_P, _P],
    "cb200_sim_mgsp_set_peers": [_P, C.POINTER(_P), C.POINTER(_P)],
    "cb200_sim_mgsp_halo_counts": [_P, C.POINTER(_I), C.POINTER(_I)],
    "cb200_trim_pool": [],
    "cb200_test_svd3": [_I, _P, _P, _P, _P, _P],
    "cb200_test_stress": [_I, _I, ParticleBuffer, _I, _P, _P, _P, _P, _P, _P],
    "cb200_sim_profile": [_P, _I],
    "cb200_sim_profile_read": [_P, C.POINTER(C.c_double), C.POINTER(_I)],
    "cb200_sim_profile_phases": [_P, C.POINTER(C.c_double)],
}


def lib():
    """Load libclaymore_b200.so.  Raises CB200Error when it has not been built: there is no fallback path."""
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB):
            raise CB200Error(f"{_LIB} not found: build it with claymore_b200.build_library() / __graft_entry__.build() (nvcc, sm_90a). "
                             "claymore_b200 has no CPU fallback.")
        L = C.CDLL(_LIB)
        for name, args in _SIGNATURES.items():
            fn = getattr(L, name, None)
            if fn is None:
                raise CB200Error(f"{_LIB} does not export {name}: rebuild it (claymore_b200.build_library(force=True))")
            fn.argtypes = args
            fn.restype = C.c_int
        L.cb200_sim_launch_count.argtypes = [_P]
        L.cb200_sim_launch_count.restype = C.c_longlong
        if hasattr(L, "cb200_default_material"):
            L.cb200_default_material.argtypes = [_CFG, _I, C.POINTER(ParticleBuffer)]
            L.cb200_default_material.restype = None
        L.cb200_version.restype = C.c_char_p
        L.cb200_error_string.restype = C.c_char_p
        L.cb200_error_string.argtypes = [_I]
        _lib = L
    return _lib


def check(err, what=""):
    if err != 0:
        msg = lib().cb200_error_string(err).decode()
        raise CB200Error(f"{what}: CUDA error {err} ({msg})")
