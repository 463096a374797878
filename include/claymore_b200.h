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
 *                    (cellbuckets: cell-major rows, slot s of cell c of block b at (b*64 + c)*max_ppc + s; the step
 *                    driver's internal cell buckets group the slots by eight instead and are not visible through the ABI)
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

/* Analytic collision objects (DESIGN.md section 2.9): closed-form shapes with the collider's boundary types and motion model,
 * up to CB200_MAX_COLLISION_OBJECTS per simulator, no device memory.  A shape is defined in the collider's material space, the
 * point x = R(t)^T (node dx - trans - trans_vel t) / (1 + dsdt t) * scale + trans that the level-set collider queries (R(t) =
 * rot_mat Rx(omega_x t) Ry(omega_y t) Rz(omega_z t)); for a static object (rot_mat = I, scale 1, no velocities) that is world
 * space.  The shape vectors a and b:
 *   CB200_SHAPE_PLANE     a = a point p, b = the normal n (made unit length in double): solid where (x - p) . n <= 0, normal n
 *   CB200_SHAPE_BOX       a = lo, b = hi, axis-aligned: solid where lo <= x <= hi; normal of the nearest face (largest
 *                         max(lo_d - x_d, x_d - hi_d), ties to the lowest axis; -1 towards lo only where strictly nearer)
 *   CB200_SHAPE_SPHERE    a = centre c, b[0] = radius r: solid where |x - c|^2 <= r^2; normal (x - c) / |x - c|, 0 at c
 *   CB200_SHAPE_CYLINDER  a = centre c, b[0] = radius r, b[1] = half height h, axis along material-space y (orient it with
 *                         rot_mat), capped: solid where (x-c)_x^2 + (x-c)_z^2 <= r^2 and |(x-c)_y| <= h; normal +-y when
 *                         h - |(x-c)_y| < r - rho, else radial (0 on the axis)
 * type and friction act as the level-set collider's (a zero normal: SEPARATE sets v to 0, SLIP leaves it).  Unused b
 * components are ignored. */
enum { CB200_SHAPE_PLANE = 0, CB200_SHAPE_BOX = 1, CB200_SHAPE_SPHERE = 2, CB200_SHAPE_CYLINDER = 3 };
#define CB200_MAX_COLLISION_OBJECTS 16
typedef struct cb200_collision_object {
	int shape, type;
	float friction;
	float a[3], b[3];
	float rot_mat[9];
	float trans[3], trans_vel[3], omega[3];
	float dsdt, scale;
} cb200_collision_object;

/* The grid update with the level-set collider `collider` (NULL: none) and then the n objects objs[0, n) in list order, all placed
 * at `time`.  n = 0 runs exactly cb200_update_grid_velocity_query_max (collider NULL) or ..._collider.  cudaErrorInvalidValue
 * for an invalid object (see cb200_sim_set_collision_objects) or collider. */
CB200_API int cb200_update_grid_velocity_query_max_objects(const cb200_config* cfg, int block_count, float* grid, cb200_partition partition, float dt, const cb200_collider* collider, const cb200_collision_object* objs, int n, float time, float* max_vel, void* stream);

/* Level-set collision objects (DESIGN.md section 2.11): CB200_SHAPE_LEVELSET, a level set from an SDFGen `.sdf` file evaluated in the
 * object's material space, in the same list as the analytic shapes and with their types, friction and motion.  Only the file's lattice
 * is stored on the device: one float4 per node (phi, g_i, g_j, g_k), SDFGen order (i fastest), g the central difference of phi in
 * index units, 0.5f * (phi[i+1] - phi[i-1]) in float32, one-sided (phi[1] - phi[0], phi[n-1] - phi[n-2]) on the lattice faces.
 *   CB200_SHAPE_LEVELSET  a = the material-space position of node (0, 0, 0), b[0] = node spacing c > 0, b[1] = the index of the
 *                         level set in the simulator's registry (an exact integer in [0, count)); b[2] is ignored.
 * At the material-space point x: q_d = (x_d - a_d) / c (a true division); outside [0, n_d - 1] on any axis no hit; else
 * i0 = min(floor(q), n - 2), t = q - i0, and the four channels are interpolated trilinearly (the dense collider's corner order).  Solid
 * where phi <= 0; normal the interpolated g, normalised only when |g|^2 > 0 (a zero normal acts as for the other shapes).  The wall
 * band does not apply. */
enum { CB200_SHAPE_LEVELSET = 4 };
#define CB200_MAX_COLLISION_LEVELSETS 16
/* one prepared lattice on the device: lattice = float4[ni nj nk] (as float[4 ni nj nk]) */
typedef struct cb200_levelset {
	const float* lattice;
	int ni, nj, nk;
} cb200_levelset;
/* Builds the device lattice (float[4 ni nj nk]) from the DEVICE phi (float[ni nj nk]) of `header`.  cudaErrorInvalidValue for a
 * dimension below 2, ni nj nk >= 2^31 or a null pointer. */
struct cb200_sdf_header; /* below, with the .sdf sampler */
CB200_API int cb200_levelset_prepare(const struct cb200_sdf_header* header, const float* phi, float* lattice, void* stream);
/* cb200_update_grid_velocity_query_max_objects where objs may hold CB200_SHAPE_LEVELSET entries, whose b[1] indexes
 * levelsets[0, n_levelsets) (at most CB200_MAX_COLLISION_LEVELSETS prepared lattices). */
CB200_API int cb200_update_grid_velocity_query_max_levelsets(const cb200_config* cfg, int block_count, float* grid, cb200_partition partition, float dt, const cb200_collider* collider, const cb200_collision_object* objs, int n, const cb200_levelset* levelsets, int n_levelsets, float time, float* max_vel, void* stream);
/* The boundary impulse report (DESIGN.md section 2.13).  Body 0 is the level-set collider (all zeros without one), body 1 + i is
 * object i of the list (analytic or CB200_SHAPE_LEVELSET); sinks and the wall band are not bodies.  Per body and grid update:
 *   J = sum m (v_in - v_out)                 over the nodes with mass,
 *   L = sum (p - b(t)) x m (v_in - v_out),   p = n dx the node, b(t) = trans + trans_vel t the pivot the body's omega turns about,
 * v_in the velocity the body receives in the chain (after the wall mask, gravity and every earlier body), v_out the one it leaves.
 * A row is (Jx, Jy, Jz, Lx, Ly, Lz); a body that changes no node's velocity reports exactly 0.  Mean force over a span of simulated
 * time is J / span, mean torque L / span. */
#define CB200_FORCE_COMPONENTS 6
/* cb200_update_grid_velocity_query_max_levelsets that also ADDS each body's (J, L) of this grid update into the DEVICE
 * impulses[(1 + n) * CB200_FORCE_COMPONENTS] (double).  The velocities and the max are those of the entry without the report.
 * cudaErrorInvalidValue, nothing launched, for a null impulses or what that entry rejects. */
CB200_API int cb200_update_grid_velocity_query_max_forces(const cb200_config* cfg, int block_count, float* grid, cb200_partition partition, float dt, const cb200_collider* collider, const cb200_collision_object* objs, int n, const cb200_levelset* levelsets, int n_levelsets, float time, float* max_vel, double* impulses, void* stream);

/* Motion tracks of collision objects (DESIGN.md section 2.14): keyframed poses the grid update evaluates at the sub-step's time.
 * A key is (t, pos, rot): the simulated time, where the object's pivot is then and a unit quaternion rot = (w, x, y, z) (normalised in
 * double by cb200_track_prepare).  A track holds 1 to CB200_MAX_TRACK_KEYS keys with strictly increasing t; flags is
 * CB200_TRACK_LINEAR or CB200_TRACK_SMOOTH, optionally | CB200_TRACK_PERIODIC.
 *   position c(t): LINEAR piecewise linear; SMOOTH cubic Hermite with tangents m_k = (c_{k+1} - c_{k-1}) / (t_{k+1} - t_{k-1}),
 *                  one-sided at the ends (a PERIODIC track's wrap around: the last key is the first);
 *   rotation Q(t): consecutive quaternions are aligned to one hemisphere; segment k is q_k (x) exp(u theta_k a_k / 2),
 *                  u = (t - t_k) / (t_{k+1} - t_k), so the world angular velocity R(q_k) a_k theta_k / (t_{k+1} - t_k) is constant on it;
 *   outside: before the first key the first pose, from the last key on the last pose, both at rest; PERIODIC maps t >= t_last to
 *            t_0 + fmodf(t - t_0, t_last - t_0) (float) first.
 * The object's pivot is c(t) and its rotation Q(t) R0 (R0 its rot_mat): its material-space point is R(t)^T (p - c(t)) scale + trans and
 * its velocity the rigid c'(t) + omega(t) x (p - c(t)); the force report's torque is about c(t).  A tracked object must have
 * trans_vel = omega = 0 and dsdt = 0.  Rejected (cudaErrorInvalidValue, nothing changed): keys not strictly increasing, a non-finite
 * value, a zero quaternion, neighbouring quaternions exactly 180 degrees apart (q_k . q_{k+1} = 0), a PERIODIC track with fewer than 2
 * keys or whose last pose differs from its first (quaternions equal up to sign), more than CB200_MAX_TRACK_KEYS keys, unknown flags. */
typedef struct cb200_track_key {
	float t;
	float pos[3];
	float rot[4];
} cb200_track_key;
enum { CB200_TRACK_LINEAR = 0, CB200_TRACK_SMOOTH = 1, CB200_TRACK_PERIODIC = 2 };
#define CB200_MAX_TRACK_KEYS 4096
/* one prepared key (64 B): the key's t and pos, its hemisphere-aligned unit quaternion, the position tangent m_k (SMOOTH; 0 for
 * LINEAR) and the rotation vector theta_k a_k of the segment it starts (0 on the last key) */
typedef struct cb200_track_record {
	float t;
	float pos[3];
	float rot[4];
	float tangent[3];
	float rotvec[3];
	float reserved[2];
} cb200_track_record;
/* object i's records: table[offset, offset + count); count 0: not tracked */
typedef struct cb200_track_span {
	int offset, count, flags;
} cb200_track_span;
/* Host only: validates keys[0, n) with flags (the rejections above) and writes n records to out.  cudaErrorInvalidValue, out
 * untouched, on a rejection or a null pointer. */
CB200_API int cb200_track_prepare(const cb200_track_key* keys, int n, int flags, cb200_track_record* out);
/* cb200_update_grid_velocity_query_max_forces (impulses may be NULL: no report) where object i with spans[i].count > 0 moves on its
 * track: records is the DEVICE table the spans index (prepared by cb200_track_prepare), spans a HOST array of n.  Allocates nothing.
 * cudaErrorInvalidValue, nothing launched, for what that entry rejects, a null spans, a span with count < 0, count >
 * CB200_MAX_TRACK_KEYS, offset < 0 or unknown flags, a tracked object with trans_vel, omega or dsdt set, or a null records. */
CB200_API int cb200_update_grid_velocity_query_max_tracks(const cb200_config* cfg, int block_count, float* grid, cb200_partition partition, float dt, const cb200_collider* collider, const cb200_collision_object* objs, int n, const cb200_levelset* levelsets, int n_levelsets, const cb200_track_record* records, const cb200_track_span* spans, float time, float* max_vel, double* impulses, void* stream);

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
/* update_{fr,j_fluid,nacc}_parameters  gmpm_simulator.cuh:211-254 (sand: defaults as in gmpm.cu:134-135, or this call).
 * Each may also be called between sub-steps of a set-up simulator: the change applies from the next sub-step, in graph and
 * stream mode alike (the call synchronises and re-captures the sub-step graphs).  The clock and the force report are kept.
 * Under MGSP every rank that holds the model must make the same call before its next step.  A wrong material for the model,
 * a model index out of range or no model at all is refused (cudaErrorInvalidValue) and changes nothing. */
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
/* output_model  gmpm_simulator.cuh:594-634: positions to HOST float[3*n]; returns count in *n_out.  Rows in the order of a
 * checkpoint of the same state (partition order, then bucket order), bit for bit the first three columns of its state rows
 * and of cb200_sim_particle_state; two calls on an unchanged simulator return the same bytes */
CB200_API int cb200_sim_retrieve(cb200_sim* sim, int model, float* positions_host, int* n_out);
/* same, zero-copy: *positions_pinned is the simulator's pinned staging buffer, valid until the next retrieve of that model */
CB200_API int cb200_sim_retrieve_pinned(cb200_sim* sim, int model, const float** positions_pinned, int* n_out);
/* full particle state (all channels, [n][channels]) to HOST: byte for byte the model's section of a checkpoint of the same
 * state (a particle the partition lost is a row of zeros in both) */
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
/* Replaces the simulator's analytic collision objects by objs[0, n) (n = 0 clears them).  Every entry is checked first: an
 * unknown shape or type, scale 0, a non-finite value, a zero plane normal, lo > hi, a radius or half height <= 0 or n outside
 * [0, CB200_MAX_COLLISION_OBJECTS] return cudaErrorInvalidValue with the simulator unchanged.  Each sub-step's grid update
 * resolves the level-set collider first, then the objects in list order (overlapping objects depend on that order), all placed
 * at the simulated time at the start of the sub-step.  Synchronises and re-captures the sub-step graphs; call it between
 * sub-steps.  Objects are scene input: a checkpoint does not store them, set them before cb200_sim_restore. */
CB200_API int cb200_sim_set_collision_objects(cb200_sim* sim, const cb200_collision_object* objs, int n);
/* Moves collision object `object` (an index into the list cb200_sim_set_collision_objects set) along keys[0, n) with flags (the
 * semantics of cb200_track_key); n = 0 clears its track.  The simulator keeps the prepared keys of all its tracks, at most
 * CB200_MAX_TRACK_KEYS together, on the device.  cudaErrorInvalidValue, nothing changed, for what cb200_track_prepare rejects, an
 * object index outside the list, a tracked object with trans_vel, omega or dsdt set, or a total above CB200_MAX_TRACK_KEYS.
 * The grid update, the MGSP carry predictor and the set-up predictor evaluate the track at the time they place objects at.  Resets
 * the force report.  Synchronises and re-captures the sub-step graphs; call it between sub-steps.  Replacing the object list clears
 * every track.  Tracks are scene input, as objects are: a checkpoint does not store them; under MGSP set the same on every rank. */
CB200_API int cb200_sim_set_object_track(cb200_sim* sim, int object, const cb200_track_key* keys, int n, int flags);
/* Registers a level set for CB200_SHAPE_LEVELSET objects and sinks: phi_host (ni nj nk floats of `header`) is uploaded, its lattice
 * prepared on the device (16 B per node, kept until cb200_sim_destroy or cb200_sim_clear_collision_levelsets) and its index written to
 * *id.  cudaErrorInvalidValue, nothing changed, for a bad header (as cb200_sdf_parse), a null pointer or a full registry
 * (CB200_MAX_COLLISION_LEVELSETS).  Level sets are scene input, as objects are: register them before cb200_sim_restore.  Both calls
 * synchronise and re-capture the sub-step graphs. */
CB200_API int cb200_sim_add_collision_levelset(cb200_sim* sim, const struct cb200_sdf_header* header, const float* phi_host, int* id);
/* Frees every registered level set; cudaErrorInvalidValue, nothing changed, while a set collision object refers to one. */
CB200_API int cb200_sim_clear_collision_levelsets(cb200_sim* sim);
/* simulated time since initial_setup: the sum of the dt of every finished sub-step (synchronises) */
CB200_API int cb200_sim_time(cb200_sim* sim, double* time);
/* Turns the boundary impulse report (cb200_update_grid_velocity_query_max_forces) of every sub-step's grid update on (enable != 0) or
 * off, and resets its accumulator.  Off (the default) the grid update is the one without the report.  Synchronises and re-captures
 * the sub-step graphs; call it between sub-steps. */
CB200_API int cb200_sim_set_force_report(cb200_sim* sim, int enable);
/* Copies the report accumulated since its last reset, n_bodies = 1 + the number of collision objects rows of (Jx, Jy, Jz, Lx, Ly, Lz)
 * summed in double over the sub-steps, into out[capacity * CB200_FORCE_COMPONENTS], the simulated time those sub-steps cover into
 * *elapsed, then resets it.  Synchronises.  cudaErrorInvalidValue, nothing written or reset, when the report is off, for a null
 * pointer or for capacity < 1 + the number of objects.  cb200_sim_set_force_report, cb200_sim_set_collider,
 * cb200_sim_clear_collider, cb200_sim_set_collision_objects and a restore reset it as well (the rows change meaning); adding or
 * removing particles keeps it; a checkpoint does not store it.  Under MGSP each rank reports the blocks it is the lowest rank to hold: the ranks' rows sum to the whole. */
CB200_API int cb200_sim_collision_forces(cb200_sim* sim, double* out, int capacity, int* n_bodies, double* elapsed);
/* number of kernels this library launched on behalf of `sim` since creation */
CB200_API long long cb200_sim_launch_count(cb200_sim* sim);

/* ------------------------------------------------------------------------------------------------
 * Checkpoint / restore of a running simulation at a sub-step boundary.  The checkpoint holds the physical state, not the
 * device containers, so it restores into a simulator of any block capacity, graph mode or auto_grow setting.
 *
 * Blob layout (all little-endian; every offset and size is a 64-bit byte count from the start of the blob):
 *   header, CB200_CHECKPOINT_HEADER_BYTES (1024) bytes:
 *     0 char[8] "CB200CKP" | 8 u32 version | 12 u32 n_models (1..8) | 16 u64 bytes (whole blob)
 *     24 cb200_config (i32 domain_bits, i32 max_ppc, i32 boundary, f32 gravity, f32 cfl)
 *     44 f32 dt_default | 48 i32 fps | 52 i32 mgsp_rank | 56 i32 mgsp_world | 60 i32 error bits
 *     64 f32 dt | 68 f32 next_dt | 72 f32 step_time | 76 f32 frame_time | 80 f64 sim_time | 88 i64 steps
 *     96 i64 frames (finished by cb200_sim_advance_frame) | 104 i32 pbc | 108 i32 nbc | 112 i32 ebc | 116 i32 max_blocks at save
 *     120 u64 keys_offset | 128 u64 keys_bytes | 136 u64 grid_offset | 144 u64 grid_bytes | 152..255 zero
 *     256 + 96 m, m < 8: table of contents entry of model m (zero when m >= n_models):
 *       0 i32 material | 4 i32 channels (4 / 12 / 13) | 8 i64 count | 16 u64 offset | 24 u64 bytes (= count * channels * 4)
 *       32 sixteen 4-byte parameters in cb200_particle_buffer order, rho .. hardening_on
 *   data sections (written 256-byte aligned, in this order; a reader must use the offsets):
 *     per model: float state[count][channels], the layout of cb200_sim_particle_state
 *     int32 keys[nbc][3]: the grid blocks of grid[0] (particle blocks first)
 *     float grid[nbc][256]: mass and momentum the next sub-step's grid update starts from, layout of a grid block
 * Particle rows are in partition order, then bucket order inside a block: two checkpoints of an unchanged simulator are
 * byte-identical.  The collider field and the collision objects are not stored: set them before cb200_sim_restore. */
#define CB200_CHECKPOINT_VERSION 1
#define CB200_CHECKPOINT_HEADER_BYTES 1024
typedef struct cb200_checkpoint_model {
	int material;
	int channels;
	long long count;
	unsigned long long offset, bytes;
	cb200_particle_buffer params; /* pointers are null */
} cb200_checkpoint_model;
typedef struct cb200_checkpoint_info {
	unsigned int version;
	int n_models;
	unsigned long long bytes;
	cb200_config cfg;
	float dt_default;
	int fps, mgsp_rank, mgsp_world;
	int error;
	float dt, next_dt, step_time, frame_time;
	double sim_time;
	long long steps, frames;
	int particle_block_count, neighbor_block_count, exterior_block_count, max_blocks;
	unsigned long long keys_offset, keys_bytes, grid_offset, grid_bytes;
	cb200_checkpoint_model models[8];
} cb200_checkpoint_info;
/* Host only, needs no device: validates a blob and fills *info.  cudaErrorInvalidValue for a bad magic or version, a blob shorter
 * or longer than its header says, sections that overlap the header or each other or run past `bytes`, section sizes that disagree
 * with count x channels or nbc, more than 8 (or no) models, a material out of range, counts that are not 0 < count < 2^31 and
 * 0 < pbc <= nbc <= ebc, and keys outside the domain or repeated. */
CB200_API int cb200_checkpoint_inspect(const void* blob, size_t bytes, cb200_checkpoint_info* info);
/* Snapshot at the current sub-step boundary, enqueued on the simulator's stream; waits for the snapshot kernel (not for the sub-steps
 * queued after it), then queues the copy into a pinned buffer the simulator owns on a stream of its own and returns.  *bytes: size
 * of the blob.  Sub-steps enqueued afterwards overlap with the copy.  Format version 1 holds no empty model: while a model has no
 * particle (after cb200_sim_remove_particles / _rows took them all) it returns cudaErrorNotSupported and changes nothing. */
CB200_API int cb200_sim_checkpoint_begin(cb200_sim* sim, size_t* bytes);
/* waits for the copy of the last begin; *blob_pinned stays valid until the next begin, reserve or destroy */
CB200_API int cb200_sim_checkpoint_end(cb200_sim* sim, const void** blob_pinned, size_t* bytes);
/* In place of init_model + initial_setup on a freshly created simulator (no models): rebuilds the partition, bins and buckets from the
 * saved particles, the grid from the saved blocks and the step clock from the saved one.  cudaErrorInvalidValue (simulator unchanged)
 * for a blob inspect rejects, a simulator that has models or is set up, or a cb200_config, dt_default, fps, mgsp_rank or mgsp_world
 * that differs from the simulator's; cudaErrorMemoryAllocation (unchanged) when max_blocks is below the saved ebc.  A blob that
 * passes inspect but whose particles or keys do not rebuild the saved partition returns cudaErrorIllegalState without writing out of
 * bounds; such a simulator can only be destroyed.
 * restore = restore_models + initial_setup.  restore_models takes the place of init_model: it checks the blob as above, registers
 * the saved models and stages their state on the device (it allocates, so it synchronises the device); the next initial_setup
 * restores instead of rasterising.  MGSP ranks that share a device in one process call restore_models on every rank, wire the
 * peers, then run initial_setup concurrently, as after init_model.  The first checkpoint_begin allocates a pinned buffer: in that
 * configuration take it while no rank has sub-steps in flight. */
CB200_API int cb200_sim_restore_models(cb200_sim* sim, const void* blob_host, size_t bytes);
CB200_API int cb200_sim_restore(cb200_sim* sim, const void* blob_host, size_t bytes);

/* ------------------------------------------------------------------------------------------------
 * Per-frame particle output (output_model, gmpm_simulator.cuh:594-634, and the IO thread of Library/MnSystem/IO/IO.h): one
 * point-only BGEO V5 file per model, byte-identical to what partio's writer produces for the same points.  A point record is
 * x y z 1.0, then v (VECTOR 3) if CB200_OUTPUT_V, then J (FLOAT 1) if CB200_OUTPUT_J, every word big-endian; after the records come
 * the bytes 0x00 0xff.  Rows are in the checkpoint's order (partition order, then bucket order).  v is the G2P of grid[0]'s node
 * velocities at the particle (MLS-MPM keeps no particle velocity); J is the fluid's J or det F.
 * ---------------------------------------------------------------------------------------------- */
#define CB200_OUTPUT_V 1u
#define CB200_OUTPUT_J 2u
/* returned when a file could not be opened or written; the errno comes with cb200_sim_frame_output_wait */
#define CB200_ERROR_OUTPUT_IO 2000
/* Host only: the header of a file of `points` points (0 <= points < 2^31) with `attributes`, and the 2-byte trailer.  *bytes gets
 * the size; cudaErrorInvalidValue for a point count or attribute bits out of range, or a capacity below the size. */
CB200_API int cb200_bgeo_header(long long points, unsigned attributes, void* out, size_t capacity, size_t* bytes);
CB200_API int cb200_bgeo_trailer(void* out, size_t capacity, size_t* bytes);
/* Writes the particles of every model at the current sub-step boundary to paths[m] (one path per model).  Runs the scans and the
 * gather on the simulator's stream and waits for the gather only (the headers need the counts), queues the copy into a pinned
 * buffer on a stream of its own and hands the files to a writer thread the simulator owns, then returns: sub-steps issued
 * afterwards overlap with the copy and the writes.  One frame is in flight at a time: a call made while the previous frame's files
 * are still being written waits for them first.  The staging and pinned buffers are allocated on first use and reused.
 * cudaErrorInvalidValue (nothing queued, simulator usable) for a simulator not set up, a null path or unknown attribute bits;
 * CB200_ERROR_OUTPUT_IO (nothing queued) while a failed write of an earlier frame has not been collected by frame_output_wait. */
CB200_API int cb200_sim_frame_output(cb200_sim* sim, const char* const* paths, unsigned attributes);
/* Waits until every queued file is written.  When an open or write failed, returns CB200_ERROR_OUTPUT_IO with its errno in
 * *os_errno (nullable) and clears it; a partially written file is removed.  0 and *os_errno = 0 otherwise. */
CB200_API int cb200_sim_frame_output_wait(cb200_sim* sim, int* os_errno);
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
 * Particle models sampled from a level set (the reference's read_sdf, Library/MnSystem/IO/ParticleIO.hpp:65-97, and
 * SampleGenerator::LoadSDF / GenerateUniformSamples, Library/MnSystem/IO/PoissonDisk/SampleGenerator.h:68-93,149-177; gmpm.cu:152-159
 * builds every model so).  The file is SDFGen text: `ni nj nk`, `min_x min_y min_z`, `h`, then ni nj nk values with i fastest
 * (phi[i + ni (j + nj k)]).  The origin is metadata only.  Placement: one scale for all axes, c = h min_d span_d / ((n_d - 1) h);
 * node q (index units) lands at offset + q c, and the node box [offset, offset + (n - 1) c] must lie inside [0, 1]^3.
 *   CB200_SDF_RANDOM   the reference's sampler with DESIGN §2.7's S1-S4 fixed: valid cells (a negative node) in ascending id
 *                      i + (ni-1)(j + (nj-1) k); spc = ppc (c / dx)^3; valid cell v holds candidates floor(v spc) <= j <
 *                      floor((v + 1) spc); candidate j draws Philox4x32-10 at counter (j lo, j hi, 0, 0), key (seed lo, seed hi), and
 *                      u_d = (r_d >> 8) 2^-24 from the first three words; q = cell + u is kept when the trilinear phi (double,
 *                      fetchGridTrilinear's corners and order) is negative.  Expected density: ppc particles per simulation cell.
 *   CB200_SDF_LATTICE  ppc = k^3 (k = 1..4) lattice points per simulation cell, (cell + (m - (k-1)/2) / k) dx, cells row-major with x
 *                      slowest, kept where q = (x - offset) / c lies in [0, n - 1] and phi(q) < 0 (samplers.uniform_box's order
 *                      and bits for k = 2).
 * Positions are offset + q c in double rounded to float32, in candidate (lattice point) order.
 * ---------------------------------------------------------------------------------------------- */
typedef struct cb200_sdf_header {
	int ni, nj, nk;  /* nodes per axis */
	float min[3];    /* SDFGen's origin (not used for placement) */
	float h;         /* node spacing */
} cb200_sdf_header;
#define CB200_SDF_RANDOM 0
#define CB200_SDF_LATTICE 1
typedef struct cb200_sdf_sampling {
	int mode;                /* CB200_SDF_RANDOM / CB200_SDF_LATTICE */
	int ppc;                 /* particles per simulation cell (lattice: 1, 8, 27 or 64) */
	double offset[3];        /* world position of node 0 */
	double span[3];          /* the box the level set is fitted into (the smallest ratio decides) */
	unsigned long long seed; /* random: Philox key */
} cb200_sdf_sampling;
/* Host only.  Parses `bytes` of text with strtof, so values are bitwise those of LoadSDF's `>>`.  phi (nullable): receives the
 * ni nj nk values when capacity allows.  cudaErrorInvalidValue for a dimension below 2 or ni nj nk >= 2^31, an h that is not finite
 * and positive, a value that is not a finite number, too few or too many values, or a capacity below ni nj nk. */
CB200_API int cb200_sdf_parse(const char* text, size_t bytes, cb200_sdf_header* header, float* phi, size_t capacity);
/* Samples on the current device (phi_host: ni nj nk floats) and returns the particle count in *n_out; with pos_host (nullable)
 * and capacity >= the count (in particles) the positions are copied there.  Synchronises `stream`.  cudaErrorInvalidValue for a
 * bad config, header, mode or ppc, a span that is not positive, a node box outside the domain, or a capacity below the count
 * (*n_out still set). */
CB200_API int cb200_sample_sdf(const cb200_config* cfg, const cb200_sdf_header* header, const float* phi_host, const cb200_sdf_sampling* sampling,
                               float* pos_host, long long capacity, long long* n_out, void* stream);
/* init_model from a level set: counts, allocates the model, then writes the positions straight into its device array.
 * cudaErrorInvalidValue, simulator unchanged, for a bad material, mode or ppc, a span that is not positive, a node box outside
 * the domain, a count of 0 or >= 2^31, a simulator that is set up or has 8 models.  *n_out (nullable): the particle count. */
CB200_API int cb200_sim_init_model_sdf(cb200_sim* sim, int material, const cb200_sdf_header* header, const float* phi_host,
                                       const cb200_sdf_sampling* sampling, const float* v0, int* model_id, int* n_out);

/* ------------------------------------------------------------------------------------------------
 * Level sets from triangle meshes (DESIGN.md section 2.12): SDFGen's make_level_set3 (Externals/SDFGen/makelevelset3.cpp:118-183)
 * on the device, bit for bit, and the lattice of SDFGen's main (main.cpp:63-118).  The result is a (cb200_sdf_header, phi) pair that
 * every .sdf consumer above takes: exact distances within exact_band cells of a triangle, fast-sweeping distances beyond, and the
 * sign by the parity of crossings along +i (a mesh that is not watertight gives streaks).
 * ---------------------------------------------------------------------------------------------- */
typedef struct cb200_mesh_header {
	int nv, nt;      /* vertices, triangles (a polygon counts as its fan) */
	float min[3];    /* the vertex bounding box (every vertex, referenced or not) */
	float max[3];
} cb200_mesh_header;
typedef struct cb200_mesh_levelset_params {
	float h;         /* node spacing, mesh units */
	int padding;     /* cells between the vertex box and the lattice's faces (below 1 means 1) */
	int exact_band;  /* 0..8: cells around each triangle's box whose distances are exact */
} cb200_mesh_levelset_params;
/* Host only.  Wavefront OBJ text: `v x y z` lines (further values ignored) and `f` lines of 3 or more references `i`, `i/t`, `i//n`
 * or `i/t/n` (1-based; negative counts back from the last vertex read); a polygon becomes the fan (v0, v_i, v_{i+1}).  Other lines
 * are ignored.  vertices (nullable): float[3 nv]; triangles (nullable): int[3 nt], 0-based; each filled when its capacity (in
 * vertices / triangles) allows.  cudaErrorInvalidValue for a `v` line without three finite numbers, an `f` line with fewer than three
 * references, a reference that is not an integer, 0, or outside the vertices, or a capacity below the count. */
CB200_API int cb200_obj_parse(const char* text, size_t bytes, cb200_mesh_header* header, float* vertices, int* triangles, size_t v_capacity,
                              size_t t_capacity);
/* The level set of HOST vertices[3 nv] / triangles[3 nt] on the current device.  *out: min = vertex box - padding h (float),
 * n_d = (unsigned) ((max_d - min_d) / h), h.  phi == NULL fills only *out, on the host.  Otherwise phi (HOST, capacity >= ni nj nk
 * floats) receives the level set, i fastest; synchronises `stream`.  cudaErrorInvalidValue, before any device work, for an h that is
 * not finite and positive, exact_band outside 0..8, no triangles, an index outside [0, nv), a non-finite vertex, any n_d < 2,
 * ni nj nk >= 2^31 or a capacity below it. */
CB200_API int cb200_mesh_levelset(const float* vertices, int nv, const int* triangles, int nt, const cb200_mesh_levelset_params* params,
                                  cb200_sdf_header* out, float* phi, size_t capacity, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Adding particles to a running simulation (sources: inlets, pouring, an object dropped later).  Both entries share one path and
 * differ only in where the candidate positions come from.  The call synchronises and acts at the current sub-step boundary.
 *   Rejections, all before anything changes (a checkpoint taken after one is byte-identical to one taken before it):
 *     cudaErrorNotSupported    MGSP mode (as cb200_sim_reserve);
 *     cudaErrorInvalidValue    a simulator that is not set up, an unknown model, unknown flag bits, a v0 that is not finite, a bad
 *                              .sdf header, mode or ppc (as cb200_sim_init_model_sdf), a candidate that is not finite or whose bucket block (cell_index - 2,
 *                              floor, per axis) lies outside the domain, a cell that would hold more than max_ppc particles
 *                              (existing ones of every model plus the new ones), or more than 2^31 - 1 particles in the model;
 *     cudaErrorMemoryAllocation  the union's exterior blocks exceed the block capacity and auto_grow is off (with auto_grow the
 *                              capacity grows, through cb200_sim_reserve, to 4/3 of them: the last step before the commit, so an
 *                              out-of-memory failure of that growth may leave the capacity grown, as cb200_sim_reserve does).
 *   n = 0, or a filter that keeps nothing, is a successful no-op.
 *   A device error after the commit has begun (out of memory while re-capturing the sub-step graphs, a failing launch) leaves a
 *   simulator that cannot step: destroy it, or restore a checkpoint into a new one.
 *   After the call, at the same boundary:
 *     - every existing particle of every model keeps all its channels bitwise (as a multiset of rows);
 *     - a new row holds the candidate's position bitwise and the model's start state: F = I (J_FLUID: J = 1), logJp = LOG_JP_0;
 *     - the partition's particle / neighbour / exterior keys are the ones initial_setup builds for the union of the positions;
 *     - grid[0] holds, cell by cell, its value before the call plus the rasterisation of the new particles (mass pb.mass, momentum
 *       mass * v0, the quadratic B-spline); blocks new to the partition hold only the new contribution;
 *     - steps, sim_time, step_time, frame_time and the frames finished are kept; dt and next_dt become min(dt, dx cfl / |v0|),
 *       initial_setup's float expression, so an emission right after initial_setup starts from the dt of a set-up over the union;
 *     - the model's bins grow to n / 32 + max_blocks; the sub-step graphs are re-captured;
 *     - every model's particle count becomes its live count: a model that lost particles before the call (kErrLostParticle,
 *       kErrCellOverflow) no longer counts them, as cb200_sim_retrieve and a checkpoint already did not.
 *   A checkpoint_begin copy or a frame_output frame in flight still delivers the state from before the call.
 * ---------------------------------------------------------------------------------------------- */
#define CB200_EMIT_EMPTY_CELLS 1u   /* keep only particles whose cell holds no particle of any model before the call */
/* Appends particles to `model` at the current sub-step boundary.  positions_host: HOST float[3n]; v0: one velocity for all of them
 * (nullable = 0).  *n_added (nullable): rows actually appended (n, or fewer with CB200_EMIT_EMPTY_CELLS).
 * CB200_EMIT_EMPTY_CELLS: a candidate's cell is cell_index(x) per axis (the cell the buckets are built by); the candidate is dropped,
 * not rejected, when any model held a particle in that cell before the call.  Candidates of one call that share a cell are all
 * kept, so emitting the same region twice at one boundary adds nothing the second time. */
CB200_API int cb200_sim_add_particles(cb200_sim* sim, int model, const float* positions_host, int n, const float* v0, unsigned flags, int* n_added);
/* The same with positions sampled on the device from a level set, as cb200_sim_init_model_sdf samples them (no host copy). */
CB200_API int cb200_sim_add_particles_sdf(cb200_sim* sim, int model, const cb200_sdf_header* header, const float* phi_host,
                                          const cb200_sdf_sampling* sampling, const float* v0, unsigned flags, int* n_added);

/* ------------------------------------------------------------------------------------------------
 * Removing particles from a running simulation (sinks: outlets, drains, discarding what leaves a region of interest).  Both entries
 * share one path and differ only in how the rows to remove are chosen.  The call synchronises and acts at the current sub-step
 * boundary.
 *   Rejections, all before anything changes (a checkpoint taken after one is byte-identical to one taken before it):
 *     cudaErrorNotSupported    MGSP mode (a rank's rebuild would have to be agreed with its peers, as for emission);
 *     cudaErrorInvalidValue    a simulator that is not set up, an empty or unknown model mask or an unknown model, unknown flag bits,
 *                              a region cb200_sim_set_collision_objects rejects, n outside [0, CB200_MAX_COLLISION_OBJECTS], a mask
 *                              length other than the model's row count, or a removal that would leave the whole simulator without
 *                              a particle.
 *   Removing nothing (n = 0, regions that hit nothing, an all-zero mask) is a successful no-op: nothing is rebuilt.
 *   A device error after the commit has begun leaves a simulator that cannot step, as for emission.
 *   After the call, at the same boundary:
 *     - every surviving particle keeps all its channels bitwise (as a multiset of rows); the removed rows are exactly those selected;
 *     - the partition's particle / neighbour / exterior keys are the ones initial_setup builds for the survivors' positions; the bins
 *       keep their capacity;
 *     - grid[0]'s mass is the survivors' rasterisation, and every node keeps the velocity it had: momentum_i = m'_i (p_i / m_i) in
 *       float32, 0 where m_i = 0.  The next sub-step reads only grid[0]'s velocities, so the survivors feel no impulse and their
 *       velocity (as cb200_sim_frame_output's v defines it) is unchanged; blocks no survivor reaches are dropped;
 *     - the whole clock is kept bitwise: dt, next_dt, steps, sim_time, step_time, frame_time, the frames finished, the error bits;
 *     - every model's particle count becomes its live count, as after an emission; the sub-step graphs are re-captured.
 *   A model may become empty: it stays registered, steps as nothing, cb200_sim_retrieve / particle_state return 0 rows, its frame
 *   files hold 0 points, and cb200_sim_add_particles* can refill it.  cb200_sim_checkpoint_begin refuses while a model is empty.
 *   A checkpoint_begin copy or a frame_output frame in flight still delivers the state from before the call.
 * ---------------------------------------------------------------------------------------------- */
#define CB200_REMOVE_OUTSIDE 1u  /* remove the particles outside the union of the regions instead of inside it */
/* Removes, from every model whose bit is set in model_mask, the particles whose position lies in any of regions[0, n): a region is a
 * cb200_collision_object (shape and motion as in section 2.9, or a registered level set as in section 2.11; type and friction are
 * ignored), placed at the simulated time, and the
 * point tested is the particle's position mapped into the object's material space as the collider maps a node.  removed[m]
 * (nullable, 8 entries): rows removed from model m. */
CB200_API int cb200_sim_remove_particles(cb200_sim* sim, unsigned model_mask, const cb200_collision_object* regions, int n,
                                         unsigned flags, long long* removed);
/* Removes the rows of `model` whose byte in remove_host[0, n) is non-zero; row i is row i of cb200_sim_retrieve / particle_state
 * at this boundary, and n must equal that row count. */
CB200_API int cb200_sim_remove_rows(cb200_sim* sim, int model, const unsigned char* remove_host, long long n, long long* removed);

/* ------------------------------------------------------------------------------------------------
 * Test-only hooks (used by tests/, not part of the drop-in surface): the device 3x3 SVD and constitutive models of g2p2g on
 * caller-supplied DEVICE vectors, against math::svd (Library/MnBase/Math/Matrix/svd.cuh:28-1124) and compute_stress<M>
 * (Projects/GMPM/constitutive_models.cuh:36-335).  F: float[9n] column-major; mode 0 = the path g2p2g takes, 1 = FIXED_COROTATED via SVD.
 * ---------------------------------------------------------------------------------------------- */
CB200_API int cb200_test_svd3(int n, const float* F, float* U, float* S, float* V, void* stream);
CB200_API int cb200_test_stress(int material, int mode, cb200_particle_buffer params, int n, const float* F_in, const float* log_jp_in, float* F_out, float* PF_out, float* log_jp_out, void* stream);
/* The step driver's bucket flatten (the rebuild's warp-per-block copy) on caller-supplied DEVICE containers of `block_count` blocks, in place
 * of cb200_cell_bucket_to_block: sizes are SET (not added to), and cell_offsets[64 * block_count] receives every cell's start in its bucket.
 * `cellbuckets` is in the reference's layout; the hook regroups it into the driver's own in a stream-ordered scratch allocation first. */
CB200_API int cb200_test_warp_flatten(const cb200_config* cfg, int block_count, const int* cell_particle_counts, const int* cellbuckets, int* particle_bucket_sizes, int* buckets, unsigned short* cell_offsets, void* stream);
/* ParticleBuffer<M> default parameters (particle_buffer.cuh:141-264) for `material` on the grid of `cfg` (pointers zero) */
CB200_API void cb200_default_material(const cb200_config* cfg, int material, cb200_particle_buffer* out);

#ifdef __cplusplus
}
#endif
#endif
