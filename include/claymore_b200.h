/*
 * claymore_b200.h -- C ABI of the H100-native MPM transfer engine (libclaymore_b200.so).
 *
 * Drop-in boundary for the fused G2P2G hot path and the sparse-grid partition/update of
 * penn-graphics-research/claymore (Projects/GMPM, Projects/MGSP).  Every entry point names the
 * reference kernel / host call it replaces (paths relative to the reference checkout).  All pointers
 * are DEVICE pointers owned by the caller unless stated otherwise; the library allocates nothing in
 * the kernel-level calls, keeps no state between them, never calls cudaSetDevice and never exits the
 * process: every function returns a cudaError_t value as int (0 == success).  `stream` is a
 * cudaStream_t passed as void*.
 *
 * Memory layouts are the reference's Structural layouts, addressed as raw pointers:
 *   particle bin   : 32 particles, SoA; channel c of bin b at  bins + b*BINF + c*32  floats,
 *                    BINF = 128 (J_FLUID, 512 B) or 512 (others, 2048 B)   particle_buffer.cuh:17-35
 *   grid block     : 4^3 cells x 4 channels SoA, 256 floats; channel c at +64*c; cell = x*16+y*4+z
 *                                                                            grid_buffer.cuh:12-14
 *   partition      : index_table int[G^3] row-major (x*G*G+y*G+z), sentinel -1; active_keys int[3*cap];
 *                    count int[1]                                            hash_table.cuh:75-135
 *   buckets        : cellbuckets/blockbuckets int[blocks*64*max_ppc]; tag = dir*(64*max_ppc) | pidib
 *                                                                            particle_buffer.cuh:134
 */
#ifndef CLAYMORE_B200_H
#define CLAYMORE_B200_H
#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define CB200_API __attribute__((visibility("default")))
#else
#define CB200_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

/* MaterialE, Projects/GMPM/settings.h:23-29 */
enum { CB200_J_FLUID = 0, CB200_FIXED_COROTATED = 1, CB200_SAND = 2, CB200_NACC = 3 };

/* runtime form of the compile-time `namespace config` (Projects/GMPM/settings.h:33-96) */
typedef struct cb200_config {
	int domain_bits; /* DOMAIN_BITS: grid is (2^bits)^3 cells, G = 2^(bits-2) blocks per axis */
	int max_ppc;     /* G_MAX_PARTICLES_IN_CELL, power of two, <= 128 */
	int boundary;    /* floor(G_BOUNDARY_CONDITION): sticky wall thickness in blocks */
	float gravity;   /* G_GRAVITY (applied to y) */
	float cfl;       /* CFL */
} cb200_config;

/* ParticleBuffer<M> passed by value in the reference (Projects/GMPM/particle_buffer.cuh:38-264) */
typedef struct cb200_particle_buffer {
	int material;
	float* bins;
	int* cell_particle_counts;
	int* particle_bucket_sizes;
	int* cellbuckets;
	int* blockbuckets;
	int* bin_offsets;
	float rho, volume, mass;
	float bulk, gamma, viscosity;         /* J_FLUID   particle_buffer.cuh:141-166 */
	float lambda, mu;                     /* FIXED_COROTATED / SAND / NACC  :168-191 */
	float cohesion, beta, yield_surface;  /* SAND  :193-224 (beta shared with NACC) */
	int volume_correction;
	float bm, xi, msqr;                   /* NACC  :226-264 */
	int hardening_on;
} cb200_particle_buffer;

/* Partition<1> passed by value in the reference (Projects/GMPM/hash_table.cuh:75-135, HaloPartition<1> :27-73) */
typedef struct cb200_partition {
	int* count;
	int* index_table;
	int* active_keys;
	int* halo_count;
	char* halo_marks;
	int* overlap_marks;
	int* halo_blocks;
} cb200_partition;

CB200_API const char* cb200_version(void);
/* device memory released by destroyed simulators is kept for re-use (per device, exact size); this returns it to the driver */
CB200_API int cb200_trim_pool(void);
CB200_API const char* cb200_error_string(int err);

/* ------------------------------------------------------------------------------------------------
 * Kernel-level entry points: one per reference kernel on the hot path; each replaces the
 * `cu_dev.compute_launch({grid, block}, kernel, args...)` call cited.
 * ---------------------------------------------------------------------------------------------- */

/* g2p2g<Partition<1>, GridBuffer, M>  Projects/GMPM/mgmpm_kernels.cuh:665-937, launched at gmpm_simulator.cuh:395 */
CB200_API int cb200_g2p2g(const cb200_config* cfg, float dt, float new_dt, int particle_block_count, cb200_particle_buffer cur, cb200_particle_buffer next, cb200_partition prev_partition, cb200_partition partition, const float* grid, float* next_grid, void* stream);

/* update_grid_velocity_query_max  mgmpm_kernels.cuh:325-420, launched at gmpm_simulator.cuh:341.  max_vel: device float, max of |v|^2 (caller zeroes it) */
CB200_API int cb200_update_grid_velocity_query_max(const cb200_config* cfg, int block_count, float* grid, cb200_partition partition, float dt, float* max_vel, void* stream);

/* Signed-distance collision object: SignedDistanceGrid (Projects/MGSP/boundary_condition.cuh:25-250).
 * sdf: DEVICE float[G^3 * 256], dense over the whole domain: one block per grid block, blocks row-major (x*G*G+y*G+z), each block
 * 4 channels SoA (signed distance, gradient x, y, z) of 64 cells (cell = x*16+y*4+z): 1 KiB per grid block.
 * rot_mat in vec3x3 storage (element (i, j) at 3*i+j); type: BoundaryT. */
enum { CB200_STICKY = 0, CB200_SLIP = 1, CB200_SEPARATE = 2 };
typedef struct cb200_collider {
	const float* sdf;
	float rot_mat[9];
	float trans[3], trans_vel[3], omega[3];
	float dsdt, scale, friction;
	int type;
} cb200_collider;

/* update_grid_velocity_query_max<Grid, Partition, Boundary>  Projects/MGSP/mgmpm_kernels.cuh:323-399, launched at
 * mgsp_benchmark.cuh:380-394: the grid update with a collider placed at `time` (the reference passes 0).  max_vel receives |v|^2,
 * half of what that kernel reports (it adds every square twice). */
CB200_API int cb200_update_grid_velocity_query_max_collider(const cb200_config* cfg, int block_count, float* grid, cb200_partition partition, float dt, const cb200_collider* collider, float time, float* max_vel, void* stream);

/* clear_grid  mgmpm_kernels.cuh:106-115 via GridBuffer::reset  grid_buffer.cuh:32-35 */
CB200_API int cb200_clear_grid(int block_count, float* grid, void* stream);

/* cell_bucket_to_block  mgmpm_kernels.cuh:70-84, launched at gmpm_simulator.cuh:429 (caller zeroes particle_bucket_sizes).
 * Order inside a block bucket is cell-major (the reference's order is atomics-dependent; any order is a valid bucket). */
CB200_API int cb200_cell_bucket_to_block(const cb200_config* cfg, int block_count, const int* cell_particle_counts, const int* cellbuckets, int* particle_bucket_sizes, int* buckets, void* stream);

/* mark_active_grid_blocks :939-952 / mark_active_particle_blocks :954-964 */
CB200_API int cb200_mark_active_grid_blocks(int block_count, const float* grid, int* marks, void* stream);
CB200_API int cb200_mark_active_particle_blocks(int block_count, const int* particle_bucket_sizes, int* marks, void* stream);

/* thrust::exclusive_scan (gmpm_simulator.cuh:257-260) and exclusive_scan_inverse (Library/MnBase/Algorithm/MappingKernels.cuh:44-55) */
CB200_API int cb200_exclusive_scan(int count, const int* in, int* out, void* stream);
CB200_API int cb200_exclusive_scan_inverse(int count, const int* map, int* map_inv, void* stream);

/* update_partition :966-977, update_buckets :979-1000, compute_bin_capacity :86-94 */
CB200_API int cb200_update_partition(const cb200_config* cfg, int block_count, const int* source_nos, cb200_partition partition, cb200_partition next_partition, void* stream);
CB200_API int cb200_update_buckets(const cb200_config* cfg, int block_count, const int* source_nos, cb200_particle_buffer pb, cb200_particle_buffer next_pb, void* stream);
CB200_API int cb200_compute_bin_capacity(int block_count, const int* particle_bucket_sizes, int* bin_sizes, void* stream);

/* register_neighbor_blocks :117-133, register_exterior_blocks :135-151 (out-of-domain keys are skipped, not UB) */
CB200_API int cb200_register_neighbor_blocks(const cb200_config* cfg, int block_count, cb200_partition partition, void* stream);
CB200_API int cb200_register_exterior_blocks(const cb200_config* cfg, int block_count, cb200_partition partition, void* stream);

/* copy_selected_grid_blocks :1002-1020 */
CB200_API int cb200_copy_selected_grid_blocks(const cb200_config* cfg, int prev_block_count, const int* prev_blockids, cb200_partition partition, const int* marks, const float* prev_grid, float* grid, void* stream);

/* Partition::reset_table  hash_table.cuh:110-112 */
CB200_API int cb200_reset_table(const cb200_config* cfg, cb200_partition partition, void* stream);

/* init-only kernels: activate_blocks :21-34, build_particle_cell_buckets :36-68, array_to_buffer :221-323,
 * rasterize :153-219, init_adv_bucket :96-104.  positions: device float[3*n] (ParticleArray, AoS xyz) */
CB200_API int cb200_activate_blocks(const cb200_config* cfg, int n, const float* positions, cb200_partition partition, void* stream);
CB200_API int cb200_build_particle_cell_buckets(const cb200_config* cfg, int n, const float* positions, cb200_particle_buffer pb, cb200_partition partition, void* stream);
CB200_API int cb200_array_to_buffer(const cb200_config* cfg, int block_count, const float* positions, cb200_particle_buffer pb, void* stream);
CB200_API int cb200_rasterize(const cb200_config* cfg, int n, const float* positions, float* grid, cb200_partition partition, float mass, const float* v0_host3, void* stream);
CB200_API int cb200_init_adv_bucket(const cb200_config* cfg, int block_count, const int* particle_bucket_sizes, int* buckets, void* stream);

/* retrieve_particle_buffer :1087-1122 (parcount: device int, caller zeroes) */
CB200_API int cb200_retrieve_particle_buffer(const cb200_config* cfg, int block_count, cb200_partition partition, cb200_partition prev_partition, cb200_particle_buffer pb, cb200_particle_buffer next_pb, float* out_positions, int* parcount, void* stream);

/* MGSP halo protocol, Projects/MGSP/halo_kernels.cuh:22-97 */
CB200_API int cb200_mark_overlapping_blocks(const cb200_config* cfg, int block_count, int otherdid, const int* incoming_block_ids, cb200_partition partition, int* count, int* out_blockids, void* stream);
CB200_API int cb200_collect_blockids_for_halo_reduction(const cb200_config* cfg, int particle_block_count, cb200_partition partition, void* stream);
CB200_API int cb200_collect_grid_blocks(const cb200_config* cfg, int count, const int* blockids, const float* grid, cb200_partition partition, float* halo_grid, void* stream);
CB200_API int cb200_reduce_grid_blocks(const cb200_config* cfg, int count, const int* blockids, float* grid, cb200_partition partition, const float* halo_grid, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Step driver: the H100-native equivalent of GmpmSimulator (Projects/GMPM/gmpm_simulator.cuh:23-786)
 * and of one MgspBenchmark device worker (Projects/MGSP/mgsp_benchmark.cuh).  Block counts, dt and
 * the step clock live on the device; a sub-step is a fixed launch sequence replayed from a CUDA graph.
 * ---------------------------------------------------------------------------------------------- */
typedef struct cb200_sim cb200_sim;

typedef struct cb200_sim_desc {
	cb200_config cfg;
	float dt_default;        /* GmpmSimulator::DEFAULT_DT / scene default_dt */
	int fps;                 /* frames per second (frame horizon for compute_dt), 0 = no frame clamp */
	int max_blocks;          /* G_MAX_ACTIVE_BLOCK */
	int use_graph;           /* 1: replay sub-steps from CUDA graphs */
	int mgsp_rank, mgsp_world; /* MGSP static partition: this shard / number of shards (1 = GMPM) */
	int mgsp_halo_cap;         /* max grid blocks shared with one peer (0 = max_blocks / 2) */
	int auto_grow;             /* 1: cb200_sim_step applies check_capacity's rule by itself (asynchronous poll every 16 sub-steps) */
} cb200_sim_desc;

typedef struct cb200_sim_stats {
	int particle_block_count, neighbor_block_count, exterior_block_count;
	int bin_count[8];
	float dt, next_dt, max_vel, step_time;
	int error;               /* 0 ok; bit0 block capacity, bit1 bin capacity, bit2 lost particle, bit3 cell overflow, bit4 MGSP halo map inconsistent */
	long long steps;
} cb200_sim_stats;

CB200_API int cb200_sim_create(const cb200_sim_desc* desc, void* stream, cb200_sim** out);
CB200_API int cb200_sim_destroy(cb200_sim* sim);
/* GmpmSimulator::init_model<M>(positions, v0)  gmpm_simulator.cuh:168-209; positions: HOST float[3*n] */
CB200_API int cb200_sim_init_model(cb200_sim* sim, int material, const float* positions_host, int n, const float* v0_host3, int* model_id);
/* update_{fr,j_fluid,nacc}_parameters  gmpm_simulator.cuh:211-254 (sand: defaults as in gmpm.cu:134-135, or this call) */
CB200_API int cb200_sim_update_fr_parameters(cb200_sim* sim, int model, float rho, float vol, float youngs, float poisson);
CB200_API int cb200_sim_update_sand_parameters(cb200_sim* sim, int model, float rho, float vol, float youngs, float poisson);
CB200_API int cb200_sim_update_j_fluid_parameters(cb200_sim* sim, int model, float rho, float vol, float bulk, float gamma, float viscosity);
CB200_API int cb200_sim_update_nacc_parameters(cb200_sim* sim, int model, float rho, float vol, float youngs, float poisson, float beta, float xi);
/* GmpmSimulator::initial_setup  gmpm_simulator.cuh:637-781 */
CB200_API int cb200_sim_initial_setup(cb200_sim* sim);
/* n sub-steps of the inner loop of main_loop (gmpm_simulator.cuh:324-580); asynchronous on the sim's stream */
CB200_API int cb200_sim_step(cb200_sim* sim, int n);
/* advance one frame like main_loop's inner for-loop (sub-steps until the frame time is reached) */
CB200_API int cb200_sim_advance_frame(cb200_sim* sim, int* steps_taken);
CB200_API int cb200_sim_sync(cb200_sim* sim);
/* GmpmSimulator::check_capacity + the resize calls of main_loop (gmpm_simulator.cuh:283-300, 371-376, 404-411, 528-548):
 * reserve grows every block-indexed container in place (contents kept, sub-step graphs re-captured); check_capacity applies
 * the reference's rule (exterior blocks > 3/4 of the capacity -> capacity x 3/2) and reports the new capacity in *grown
 * (0 = unchanged).  Both synchronise; call them between sub-steps.  Not available in MGSP mode (peer-mapped buffers). */
CB200_API int cb200_sim_reserve(cb200_sim* sim, int new_max_blocks);
CB200_API int cb200_sim_check_capacity(cb200_sim* sim, int* grown);
CB200_API int cb200_sim_capacity(cb200_sim* sim, int* max_blocks, int* grow_events);
CB200_API int cb200_sim_stats_get(cb200_sim* sim, cb200_sim_stats* out); /* synchronises */
/* output_model  gmpm_simulator.cuh:594-634: positions to HOST float[3*n]; returns count in *n_out */
CB200_API int cb200_sim_retrieve(cb200_sim* sim, int model, float* positions_host, int* n_out);
/* same, zero-copy: *positions_pinned is the simulator's pinned staging buffer, valid until the next retrieve of that model */
CB200_API int cb200_sim_retrieve_pinned(cb200_sim* sim, int model, const float** positions_pinned, int* n_out);
/* full particle state (all channels, [n][channels]) to HOST, same traversal as retrieve */
CB200_API int cb200_sim_particle_state(cb200_sim* sim, int model, float* state_host, int* n_out);
/* copies for parity checks: active keys (int[3*ebc]) and grid blocks of grid[0] (float[256*nbc]) to HOST */
CB200_API int cb200_sim_active_keys(cb200_sim* sim, int* keys_host, int capacity_blocks, int* n_out);
CB200_API int cb200_sim_grid(cb200_sim* sim, float* grid_host, int capacity_blocks, int* n_out);
/* One signed-distance collider acting on the grid update (init_boundary, mgsp_benchmark.cuh:257-266).  sdf_host: the four HOST
 * float arrays of init_from_signed_distance_file (boundary_condition.cuh:297-320) back to back -- distance, gradient x, y, z, each
 * dense row-major over the (4G)^3 grid nodes; NULL keeps the field uploaded before.  params->sdf is ignored: the simulator owns
 * the device field (G^3 KiB).  The collider is placed at the simulated time at the start of each sub-step.  Both calls
 * synchronise and re-capture the sub-step graphs; call them between sub-steps. */
CB200_API int cb200_sim_set_collider(cb200_sim* sim, const cb200_collider* params, const float* sdf_host);
CB200_API int cb200_sim_clear_collider(cb200_sim* sim);
/* simulated time since initial_setup: the sum of the dt of every finished sub-step (synchronises) */
CB200_API int cb200_sim_time(cb200_sim* sim, double* time);
/* number of kernels this library launched on behalf of `sim` since creation */
CB200_API long long cb200_sim_launch_count(cb200_sim* sim);
/* per-kernel timing for the roofline: while enabled, sub-steps are issued as plain stream launches with a
 * cudaEvent pair around every g2p2g launch; profile_read synchronises and returns the summed duration */
CB200_API int cb200_sim_profile(cb200_sim* sim, int enable);
CB200_API int cb200_sim_profile_read(cb200_sim* sim, double* g2p2g_ms_total, int* launches);
/* summed milliseconds per sub-step phase while profiling was on: out_ms[10] = {-, grid update, -, -, -, g2p2g,
 * MGSP done publish, partition rebuild, MGSP halo tagging, carry/exterior/finalize}; slots marked - stay 0 */
CB200_API int cb200_sim_profile_phases(cb200_sim* sim, double* out_ms);

/* MGSP static particle partition, one process per GPU (Projects/MGSP/mgsp_benchmark.cuh:309-559, 661-776).
 * Each rank creates its simulator with mgsp_rank / mgsp_world set and registers ITS OWN particle set with
 * init_model.  The P2G sums of halo grid blocks are bulk-add-reduced by g2p2g itself straight into the peers' next grids
 * over NVLink; the neighbour-key lists for halo tagging and max |v|^2 are exchanged by kernels that store into the peers'
 * inboxes (both CUDA IPC mapped) and publish epoch flags: the transport needs no host
 * calls per sub-step.  Setup: every rank publishes its inbox handle, all ranks open all handles (any host-side
 * all-gather: torch.distributed here), then initial_setup / step run as in the single-GPU case. */
CB200_API int cb200_sim_mgsp_inbox(cb200_sim* sim, void** inbox, void** next_grid, size_t* inbox_bytes);
/* EVERY rank must be created with the same max_blocks, mgsp_halo_cap, mgsp_world and cb200_config: the layout of the messages in a
 * peer's inbox is computed from them on both sides.  The handle blob carries them and open_peers returns cudaErrorInvalidValue on a
 * mismatch (same-process peers wired with set_peers are the caller's responsibility). */
#define CB200_MGSP_HANDLE_BYTES 160
CB200_API int cb200_sim_mgsp_ipc_handle(cb200_sim* sim, void* handle);                 /* CB200_MGSP_HANDLE_BYTES: two cudaIpcMemHandle_t (inbox, next grid) + layout words */
CB200_API int cb200_sim_mgsp_open_peers(cb200_sim* sim, const void* handles_by_rank);  /* world x CB200_MGSP_HANDLE_BYTES */
CB200_API int cb200_sim_mgsp_set_peers(cb200_sim* sim, void* const* inbox_ptrs_by_rank, void* const* next_grid_ptrs_by_rank); /* same-process peers */
/* halo statistics of the current partition (synchronises): blocks shared with each rank, halo particle blocks */
CB200_API int cb200_sim_mgsp_halo_counts(cb200_sim* sim, int* shared_blocks_by_rank, int* halo_particle_blocks);

/* ------------------------------------------------------------------------------------------------
 * Test-only hooks (used by tests/, not part of the drop-in surface): the device 3x3 SVD and constitutive models of g2p2g on
 * caller-supplied DEVICE vectors, against math::svd (Library/MnBase/Math/Matrix/svd.cuh:28-1124) and compute_stress<M>
 * (Projects/GMPM/constitutive_models.cuh:36-335).  F: float[9n] column-major; mode 0 = the path g2p2g takes, 1 = FIXED_COROTATED via SVD.
 * ---------------------------------------------------------------------------------------------- */
CB200_API int cb200_test_svd3(int n, const float* F, float* U, float* S, float* V, void* stream);
CB200_API int cb200_test_stress(int material, int mode, cb200_particle_buffer params, int n, const float* F_in, const float* log_jp_in, float* F_out, float* PF_out, float* log_jp_out, void* stream);
/* ParticleBuffer<M> default parameters (particle_buffer.cuh:141-264) for `material` on the grid of `cfg` (pointers zero) */
CB200_API void cb200_default_material(const cb200_config* cfg, int material, cb200_particle_buffer* out);

#ifdef __cplusplus
}
#endif
#endif
