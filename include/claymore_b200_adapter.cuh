// claymore_b200_adapter.cuh -- the reference-side binding of libclaymore_b200: C++ overloads with the reference's own kernel
// argument lists.
//
// A maintainer of penn-graphics-research/claymore adds this header next to Projects/GMPM/mgmpm_kernels.cuh.  It needs only the
// reference's own container headers; it unpacks the by-value containers (ParticleBuffer<M>, Partition<1>, GridBuffer,
// ParticleArray) into the POD structs of include/claymore_b200.h and forwards to the C ABI.  A call site changes from
//
//     cu_dev.compute_launch({pbc, 128}, g2p2g, dt, next_dt, cur, next, prev_partition, partition, grid, next_grid);     // gmpm_simulator.cuh:395
// to
//     mn::b200::compute_launch(cu_dev, {pbc, 128}, mn::b200::g2p2g, dt, next_dt, cur, next, prev_partition, partition, grid, next_grid);
//
// i.e. the launch shape and the argument list stay as they are.  mn::b200::compute_launch keeps the contract of
// Cuda::CudaContext::compute_launch (Library/MnSystem/Cuda/Cuda.h:151-184): arguments by value, an empty launch shape is
// a no-op, the call goes to the context's compute stream, a failure is printed and not thrown.  The launch SHAPE only carries
// the block count (the library picks its own persistent grids); kernels whose count is an explicit argument ignore it.
//
// This header is compiled against the reference by tests/test_abi_cpu.py (when /root/reference is present) and is what
// oracle/ref_gpu_driver.cu uses to swap single kernels of the reference's loop for the library's (tests/test_gpu_dropin.py).
#pragma once
#include <claymore_b200.h>

#include <MnSystem/Cuda/ExecutionPolicy.h>  // LaunchConfig

#include <array>
#include <cstdio>
#include <type_traits>

#include "grid_buffer.cuh"
#include "hash_table.cuh"
#include "particle_buffer.cuh"
#include "settings.h"

// Customisation point: how an entry point of the C ABI is reached.  Default: the linked symbol.  The test driver resolves
// the library with dlopen and routes the calls through function pointers.
// The collider overload of update_grid_velocity_query_max reaches cb200_update_grid_velocity_query_max_collider: a customised
// CB200_ADAPTER_CALL that routes that entry too defines CB200_ADAPTER_COLLIDER (with the default call it is always there).
#ifndef CB200_ADAPTER_CALL
#define CB200_ADAPTER_CALL(name) ::name
#ifndef CB200_ADAPTER_COLLIDER
#define CB200_ADAPTER_COLLIDER 1
#endif
#endif

namespace mn {
namespace b200 {

// namespace config (Projects/GMPM/settings.h:33-96) -> its runtime form
inline cb200_config config_of() {
	cb200_config c;
	c.domain_bits = config::DOMAIN_BITS;
	c.max_ppc = config::G_MAX_PARTICLES_IN_CELL;
	c.boundary = (int) config::G_BOUNDARY_CONDITION;
	c.gravity = config::G_GRAVITY;
	c.cfl = config::CFL;
	return c;
}

// ParticleBuffer<M> (particle_buffer.cuh:38-264): device pointers + material parameters
template<MaterialE M>
inline cb200_particle_buffer view(const ParticleBuffer<M>& pb) {
	cb200_particle_buffer v {};
	v.material = (int) M;
	v.bins = (float*) pb.handle.ptr;  // Instance<particle_buffer_<...>>: MemResource {void* ptr}
	v.cell_particle_counts = pb.cell_particle_counts;
	v.particle_bucket_sizes = pb.particle_bucket_sizes;
	v.cellbuckets = pb.cellbuckets;
	v.blockbuckets = pb.blockbuckets;
	v.bin_offsets = pb.bin_offsets;
	v.rho = pb.rho;
	v.volume = pb.volume;
	v.mass = pb.mass;
	if constexpr(M == MaterialE::J_FLUID) {
		v.bulk = pb.bulk;
		v.gamma = pb.gamma;
		v.viscosity = pb.viscosity;
	} else {
		v.lambda = pb.lambda;
		v.mu = pb.mu;
	}
	if constexpr(M == MaterialE::SAND) {
		v.cohesion = pb.cohesion;
		v.beta = pb.beta;
		v.yield_surface = pb.yield_surface;
		v.volume_correction = pb.volume_correction;
	}
	if constexpr(M == MaterialE::NACC) {
		v.bm = pb.bm;
		v.xi = pb.xi;
		v.beta = pb.beta;
		v.msqr = pb.msqr;
		v.hardening_on = pb.hardening_on;
	}
	return v;
}
// Partition<1> (hash_table.cuh:75-135, HaloPartition<1> :27-73)
inline cb200_partition view(const Partition<1>& p) {
	cb200_partition v {};
	v.count = p.Instance<block_partition_>::count;
	v.index_table = p.index_table;
	v.active_keys = (int*) p.active_keys;
	v.halo_count = p.halo_count;
	v.halo_marks = p.halo_marks;
	v.overlap_marks = p.overlap_marks;
	v.halo_blocks = (int*) p.halo_blocks;
	return v;
}
inline float* view(const GridBuffer& g) { return (float*) g.handle.ptr; }       // grid_buffer.cuh:16-36
inline const float* view(const ParticleArray& a) { return (const float*) a.handle.ptr; }  // AoS xyz, particle_buffer.cuh:266-271

// Cuda::CudaContext::compute_launch for library entry points (Cuda.h:151-184)
template<typename Context, typename Op, typename... Arguments>
inline void compute_launch(Context& cu_dev, LaunchConfig&& lc, Op op, Arguments... args) {
	static_assert(!std::disjunction<std::is_reference<Arguments>...>::value, "Cannot pass values to Cuda kernels by reference");
	if(lc.dg.x && lc.dg.y && lc.dg.z && lc.db.x && lc.db.y && lc.db.z) {
		const cudaError_t error = (cudaError_t) op((void*) cu_dev.stream_compute(), lc, args...);
		if(error != cudaSuccess) printf("[claymore_b200] Kernel launch failure on [COMPUTE stream] %s\n", cudaGetErrorString(error));
	}
}
// the same on an explicit stream (spare_launch, MGSP worker streams)
template<typename Op, typename... Arguments>
inline cudaError_t launch_on(cudaStream_t stream, LaunchConfig&& lc, Op op, Arguments... args) {
	if(!(lc.dg.x && lc.dg.y && lc.dg.z && lc.db.x && lc.db.y && lc.db.z)) return cudaSuccess;
	return (cudaError_t) op((void*) stream, lc, args...);
}

// ---- one functor per reference kernel; operator() takes (stream, launch shape, the reference kernel's arguments) ---------------
// g2p2g<Partition, Grid, M>  mgmpm_kernels.cuh:665-666, launched with {particle blocks, G_PARTICLE_BATCH_CAPACITY}
struct g2p2g_t {
	template<MaterialE M>
	int operator()(void* s, const LaunchConfig& lc, Duration dt, Duration new_dt, const ParticleBuffer<M> particle_buffer, ParticleBuffer<M> next_particle_buffer, const Partition<1> prev_partition, Partition<1> partition, const GridBuffer grid, GridBuffer next_grid) const {
		const cb200_config c = config_of();
		return CB200_ADAPTER_CALL(cb200_g2p2g)(&c, dt.count(), new_dt.count(), (int) lc.dg.x, view(particle_buffer), view(next_particle_buffer), view(prev_partition), view(partition), view(grid), view(next_grid), s);
	}
};
#ifdef CB200_ADAPTER_COLLIDER
// the MGSP form with a collider (Projects/MGSP/mgmpm_kernels.cuh:323-324, launched at mgsp_benchmark.cuh:380-394): Boundary is
// SignedDistanceGrid (boundary_condition.cuh:25-250), read member by member; its field is dense, so its base pointer is the
// address of block (0, 0, 0).  The reference's kernel places the collider at time 0 (:363); so does this overload.
template<typename Boundary>
inline cb200_collider collider_of(Boundary& b) {
	cb200_collider c {};
	c.sdf = &b.ch(placeholder::_0, 0, 0, 0).val_1d(placeholder::_0, 0);
	for(int i = 0; i < 3; ++i)
		for(int j = 0; j < 3; ++j) c.rot_mat[3 * i + j] = b.rot_mat(i, j);
	for(int d = 0; d < 3; ++d) {
		c.trans[d] = b.trans[d];
		c.trans_vel[d] = b.trans_vel[d];
		c.omega[d] = b.omega[d];
	}
	c.dsdt = b.dsdt;
	c.scale = b.scale;
	c.friction = b.friction;
	c.type = (int) b.type;
	return c;
}
#endif
// update_grid_velocity_query_max  :325-326; with a Boundary, the MGSP form
struct update_grid_velocity_query_max_t {
	int operator()(void* s, const LaunchConfig&, uint32_t block_count, GridBuffer grid, Partition<1> partition, Duration dt, float* max_vel) const {
		const cb200_config c = config_of();
		return CB200_ADAPTER_CALL(cb200_update_grid_velocity_query_max)(&c, (int) block_count, view(grid), view(partition), dt.count(), max_vel, s);
	}
#ifdef CB200_ADAPTER_COLLIDER
	template<typename Boundary>
	int operator()(void* s, const LaunchConfig&, uint32_t block_count, GridBuffer grid, Partition<1> partition, Duration dt, Boundary boundary, float* max_vel) const {
		const cb200_config c = config_of();
		const cb200_collider col = collider_of(boundary);
		return CB200_ADAPTER_CALL(cb200_update_grid_velocity_query_max_collider)(&c, (int) block_count, view(grid), view(partition), dt.count(), &col, 0.f, max_vel, s);
	}
#endif
};
// clear_grid  :106-107, launched with {blocks, G_BLOCKVOLUME}
struct clear_grid_t {
	int operator()(void* s, const LaunchConfig& lc, GridBuffer grid) const { return CB200_ADAPTER_CALL(cb200_clear_grid)((int) lc.dg.x, view(grid), s); }
};
// cell_bucket_to_block  :70, launched with {blocks, G_BLOCKVOLUME}
struct cell_bucket_to_block_t {
	int operator()(void* s, const LaunchConfig& lc, const int* cell_particle_counts, const int* cellbuckets, int* particle_bucket_sizes, int* buckets) const {
		const cb200_config c = config_of();
		return CB200_ADAPTER_CALL(cb200_cell_bucket_to_block)(&c, (int) lc.dg.x, cell_particle_counts, cellbuckets, particle_bucket_sizes, buckets, s);
	}
};
// compute_bin_capacity :86, init_adv_bucket :96
struct compute_bin_capacity_t {
	int operator()(void* s, const LaunchConfig&, uint32_t block_count, int const* particle_bucket_sizes, int* bin_sizes) const { return CB200_ADAPTER_CALL(cb200_compute_bin_capacity)((int) block_count, particle_bucket_sizes, bin_sizes, s); }
};
struct init_adv_bucket_t {
	int operator()(void* s, const LaunchConfig& lc, const int* particle_bucket_sizes, int* buckets) const {
		const cb200_config c = config_of();
		return CB200_ADAPTER_CALL(cb200_init_adv_bucket)(&c, (int) lc.dg.x, particle_bucket_sizes, buckets, s);
	}
};
// register_neighbor_blocks :117-118, register_exterior_blocks :135-136
struct register_neighbor_blocks_t {
	int operator()(void* s, const LaunchConfig&, uint32_t block_count, Partition<1> partition) const {
		const cb200_config c = config_of();
		return CB200_ADAPTER_CALL(cb200_register_neighbor_blocks)(&c, (int) block_count, view(partition), s);
	}
};
struct register_exterior_blocks_t {
	int operator()(void* s, const LaunchConfig&, uint32_t block_count, Partition<1> partition) const {
		const cb200_config c = config_of();
		return CB200_ADAPTER_CALL(cb200_register_exterior_blocks)(&c, (int) block_count, view(partition), s);
	}
};
// mark_active_grid_blocks :939-940, mark_active_particle_blocks :954
struct mark_active_grid_blocks_t {
	int operator()(void* s, const LaunchConfig&, uint32_t block_count, const GridBuffer grid, int* marks) const { return CB200_ADAPTER_CALL(cb200_mark_active_grid_blocks)((int) block_count, view(grid), marks, s); }
};
struct mark_active_particle_blocks_t {
	int operator()(void* s, const LaunchConfig&, uint32_t block_count, const int* particle_bucket_sizes, int* marks) const { return CB200_ADAPTER_CALL(cb200_mark_active_particle_blocks)((int) block_count, particle_bucket_sizes, marks, s); }
};
// exclusive_scan_inverse  Library/MnBase/Algorithm/MappingKernels.cuh:44-45
struct exclusive_scan_inverse_t {
	int operator()(void* s, const LaunchConfig&, int num, const int* map, int* map_inv) const { return CB200_ADAPTER_CALL(cb200_exclusive_scan_inverse)(num, map, map_inv, s); }
};
// update_partition :966-967, update_buckets :979-980
struct update_partition_t {
	int operator()(void* s, const LaunchConfig&, uint32_t block_count, const int* source_nos, const Partition<1> partition, Partition<1> next_partition) const {
		const cb200_config c = config_of();
		return CB200_ADAPTER_CALL(cb200_update_partition)(&c, (int) block_count, source_nos, view(partition), view(next_partition), s);
	}
};
struct update_buckets_t {
	template<MaterialE M>
	int operator()(void* s, const LaunchConfig&, uint32_t block_count, const int* source_nos, const ParticleBuffer<M> particle_buffer, ParticleBuffer<M> next_particle_buffer) const {
		const cb200_config c = config_of();
		return CB200_ADAPTER_CALL(cb200_update_buckets)(&c, (int) block_count, source_nos, view(particle_buffer), view(next_particle_buffer), s);
	}
};
// copy_selected_grid_blocks :1002-1003, launched with {previous neighbour blocks, G_BLOCKVOLUME}
struct copy_selected_grid_blocks_t {
	int operator()(void* s, const LaunchConfig& lc, const ivec3* prev_blockids, const Partition<1> partition, const int* marks, GridBuffer prev_grid, GridBuffer grid) const {
		const cb200_config c = config_of();
		return CB200_ADAPTER_CALL(cb200_copy_selected_grid_blocks)(&c, (int) lc.dg.x, (const int*) prev_blockids, view(partition), marks, view(prev_grid), view(grid), s);
	}
};
// init kernels: activate_blocks :21-22, build_particle_cell_buckets :36-37, array_to_buffer :221-323 ({blocks, 128}), rasterize :153-154
struct activate_blocks_t {
	int operator()(void* s, const LaunchConfig&, uint32_t particle_counts, ParticleArray particle_array, Partition<1> partition) const {
		const cb200_config c = config_of();
		return CB200_ADAPTER_CALL(cb200_activate_blocks)(&c, (int) particle_counts, view(particle_array), view(partition), s);
	}
};
struct build_particle_cell_buckets_t {
	template<MaterialE M>
	int operator()(void* s, const LaunchConfig&, uint32_t particle_counts, ParticleArray particle_array, ParticleBuffer<M> particle_buffer, Partition<1> partition) const {
		const cb200_config c = config_of();
		return CB200_ADAPTER_CALL(cb200_build_particle_cell_buckets)(&c, (int) particle_counts, view(particle_array), view(particle_buffer), view(partition), s);
	}
};
struct array_to_buffer_t {
	template<MaterialE M>
	int operator()(void* s, const LaunchConfig& lc, ParticleArray particle_array, ParticleBuffer<M> particle_buffer) const {
		const cb200_config c = config_of();
		return CB200_ADAPTER_CALL(cb200_array_to_buffer)(&c, (int) lc.dg.x, view(particle_array), view(particle_buffer), s);
	}
};
struct rasterize_t {
	int operator()(void* s, const LaunchConfig&, uint32_t particle_counts, const ParticleArray particle_array, GridBuffer grid, const Partition<1> partition, Duration, float mass, std::array<float, 3> v0) const {
		const cb200_config c = config_of();
		return CB200_ADAPTER_CALL(cb200_rasterize)(&c, (int) particle_counts, view(particle_array), view(grid), view(partition), mass, v0.data(), s);
	}
};
// retrieve_particle_buffer :1087-1088, launched with {particle blocks, 128}
struct retrieve_particle_buffer_t {
	template<MaterialE M>
	int operator()(void* s, const LaunchConfig& lc, Partition<1> partition, Partition<1> prev_partition, ParticleBuffer<M> particle_buffer, ParticleBuffer<M> next_particle_buffer, ParticleArray particle_array, int* parcount) const {
		const cb200_config c = config_of();
		return CB200_ADAPTER_CALL(cb200_retrieve_particle_buffer)(&c, (int) lc.dg.x, view(partition), view(prev_partition), view(particle_buffer), view(next_particle_buffer), (float*) view(particle_array), parcount, s);
	}
};

constexpr g2p2g_t g2p2g {};
constexpr update_grid_velocity_query_max_t update_grid_velocity_query_max {};
constexpr clear_grid_t clear_grid {};
constexpr cell_bucket_to_block_t cell_bucket_to_block {};
constexpr compute_bin_capacity_t compute_bin_capacity {};
constexpr init_adv_bucket_t init_adv_bucket {};
constexpr register_neighbor_blocks_t register_neighbor_blocks {};
constexpr register_exterior_blocks_t register_exterior_blocks {};
constexpr mark_active_grid_blocks_t mark_active_grid_blocks {};
constexpr mark_active_particle_blocks_t mark_active_particle_blocks {};
constexpr exclusive_scan_inverse_t exclusive_scan_inverse {};
constexpr update_partition_t update_partition {};
constexpr update_buckets_t update_buckets {};
constexpr copy_selected_grid_blocks_t copy_selected_grid_blocks {};
constexpr activate_blocks_t activate_blocks {};
constexpr build_particle_cell_buckets_t build_particle_cell_buckets {};
constexpr array_to_buffer_t array_to_buffer {};
constexpr rasterize_t rasterize {};
constexpr retrieve_particle_buffer_t retrieve_particle_buffer {};

}  // namespace b200
}  // namespace mn
