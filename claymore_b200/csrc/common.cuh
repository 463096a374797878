// common.cuh -- shared device-side definitions for libclaymore_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/claymore_b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "claymore_b200 kernels are written for sm_90a (H100) only"
#endif

namespace cb200 {

constexpr int kBlockVol = 64;   // 4^3 cells per grid block          (settings.h:74 G_BLOCKVOLUME)
constexpr int kBinCap = 32;     // particles per bin                 (settings.h:82 G_BIN_CAPACITY)
constexpr int kGridBlockFloats = 256;  // 4 channels x 64 cells      (grid_buffer.cuh:12)
constexpr int kMaxModels = 8;

// runtime config broadcast to kernels by value
struct Cfg {
	int domain_bits, max_ppc, boundary;
	float gravity, cfl;
	int gsize;       // blocks per axis
	int gbits;       // log2(gsize)
	int ppb;         // bucket stride per block = 64 * max_ppc
	int ppb_shift;   // log2(ppb)
	int ppc_shift;   // log2(max_ppc)
	float dx, dx_inv, d_inv;
};

inline Cfg make_cfg(const cb200_config& c) {
	Cfg k;
	k.domain_bits = c.domain_bits;
	k.max_ppc = c.max_ppc;
	k.boundary = c.boundary;
	k.gravity = c.gravity;
	k.cfl = c.cfl;
	k.gbits = c.domain_bits - 2;
	k.gsize = 1 << k.gbits;
	k.ppb = c.max_ppc * kBlockVol;
	int s = 0;
	while((1 << s) < k.ppb) ++s;
	k.ppb_shift = s;
	s = 0;
	while((1 << s) < c.max_ppc) ++s;
	k.ppc_shift = s;
	k.dx_inv = (float) (1 << c.domain_bits);
	k.dx = 1.f / k.dx_inv;
	k.d_inv = 4.f * k.dx_inv * k.dx_inv;
	return k;
}

inline bool cfg_valid(const cb200_config& c) {
	if(c.domain_bits < 4 || c.domain_bits > 10) return false;
	if(c.max_ppc < 8 || c.max_ppc > 128 || (c.max_ppc & (c.max_ppc - 1))) return false;
	if(c.boundary < 0) return false;
	return true;
}

// device views of the reference containers
struct PBuf {
	float* bins;
	int* cell_particle_counts;
	int* particle_bucket_sizes;
	int* cellbuckets;
	int* blockbuckets;
	int* bin_offsets;
};
struct Mat {
	float rho, volume, mass;
	float bulk, gamma, viscosity;
	float lambda, mu;
	float cohesion, beta, yield_surface;
	int volume_correction;
	float bm, xi, msqr;
	int hardening_on;
};
struct Part {
	int* count;
	int* table;
	int* keys;
};

inline PBuf view(const cb200_particle_buffer& b) { return PBuf {b.bins, b.cell_particle_counts, b.particle_bucket_sizes, b.cellbuckets, b.blockbuckets, b.bin_offsets}; }
inline Mat mat_of(const cb200_particle_buffer& b) { return Mat {b.rho, b.volume, b.mass, b.bulk, b.gamma, b.viscosity, b.lambda, b.mu, b.cohesion, b.beta, b.yield_surface, b.volume_correction, b.bm, b.xi, b.msqr, b.hardening_on}; }
inline Part view(const cb200_partition& p) { return Part {p.count, p.index_table, p.active_keys}; }

// A block count that is either an immediate (kernel-level ABI: the reference passes host ints) or
// device-resident (step driver: counters never leave the GPU).
struct Count {
	const int* dev;
	int imm;
	__device__ __forceinline__ int get() const { return dev ? *dev : imm; }
};
inline Count count_imm(int n) { return Count {nullptr, n}; }
inline Count count_dev(const int* p) { return Count {p, 0}; }

// Device-resident step state of the driver (replaces the host counters of GmpmSimulator,
// gmpm_simulator.cuh:104-119, and their seven D2H copies per sub-step).
struct StepState {
	int pbc, nbc, ebc;      // counts of the CURRENT partition: particle / +neighbour / +exterior blocks
	int prev_nbc;           // neighbour count of the partition the next-grid is indexed by
	int prev_ebc;
	int work_counter_mat[4];  // dynamic block queue of g2p2g, one per material launch of a sub-step (all zeroed when the state rolls)
	int error;              // sticky error bits (see cb200_sim_stats)
	float dt, next_dt;
	float max_vel_sq;       // max |v|^2 as float bits (non-negative => int compare is order preserving)
	float step_time;        // time inside the current frame
	float frame_time;       // seconds per frame (0 = no clamp)
	float dt_default;
	int bin_count[kMaxModels];
	long long steps;
	int done_counter;       // CTAs of a launch that have finished ("last CTA does the epilogue"; zero between launches)
	int frame_roll;         // cb200_sim_step with fps > 0: restart the frame clock on the device when a frame is complete (the
	                        // reference's outer frame loop, gmpm_simulator.cuh:323); 0 while cb200_sim_advance_frame drives the frames
	double sim_time;        // simulated time since initial_setup: the sum of every finished sub-step's dt (places a moving collider)
};

enum : int { kErrBlockCapacity = 1, kErrBinCapacity = 2, kErrLostParticle = 4, kErrCellOverflow = 8, kErrHaloMap = 16 };

// ------------------------------------------------------------------------------------------------
// particle channels and bins
// ------------------------------------------------------------------------------------------------
// channels of a particle: the position, then J (J_FLUID) or F (9, row-major), then logJp (SAND, NACC)
__host__ __device__ inline int ck_channels(int material) { return material == CB200_J_FLUID ? 4 : (material == CB200_FIXED_COROTATED ? 12 : 13); }
// floats of one bin of kBinCap particles (J_FLUID: 4 channels, the others: 16)
__host__ __device__ constexpr int bin_floats(int material) { return material == CB200_J_FLUID ? 128 : 512; }
// particle i of the bucket whose bins start at bin `first`: its channel c is at [c * kBinCap]
template<class T>
__device__ __forceinline__ T* bin_slot(T* bins, int first, int i, int binf) { return bins + ((size_t) first + (i >> 5)) * binf + (i & 31); }

// The start state of a particle at x (array_to_buffer, mgmpm_kernels.cuh:221-323), channel c to out[c * stride]: the position, then
// J = 1 or F = I, then logJp = ParticleBuffer<M>::LOG_JP_0 (particle_buffer.cuh:207, 241)
__device__ __forceinline__ void start_state(int material, const float* x, float* out, int stride) {
	out[0] = x[0];
	out[stride] = x[1];
	out[2 * stride] = x[2];
	if(material == CB200_J_FLUID) {
		out[3 * stride] = 1.f;
		return;
	}
#pragma unroll
	for(int d = 0; d < 9; ++d) out[(3 + d) * stride] = (d % 4 == 0) ? 1.f : 0.f;
	if(material == CB200_SAND) out[12 * stride] = 0.f;
	if(material == CB200_NACC) out[12 * stride] = -0.01f;
}

// ------------------------------------------------------------------------------------------------
// index helpers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool in_domain(const Cfg& c, int x, int y, int z) { return ((unsigned) x < (unsigned) c.gsize) & ((unsigned) y < (unsigned) c.gsize) & ((unsigned) z < (unsigned) c.gsize); }
__device__ __forceinline__ int table_offset(const Cfg& c, int x, int y, int z) { return (((x << c.gbits) + y) << c.gbits) + z; }
__device__ __forceinline__ int table_query(const Cfg& c, const int* __restrict__ table, int x, int y, int z) { return in_domain(c, x, y, z) ? __ldg(table + table_offset(c, x, y, z)) : -1; }
// Slot `slot` of cell `cell` of block `block` in the step driver's cell buckets.  The reference's rows ((block * 64 + cell) * max_ppc
// + slot) are kept by the kernel-level ABI; the driver groups slots by eight inside each block's ppb slice, [max_ppc / 8][64 cells][8],
// so that slots 0-7 of all 64 cells of a block (every tag of a block whose cells hold at most eight) are 2 KiB of contiguous memory,
// and one warp load of the flatten (eight slots of four cells) is one 128-byte line.  max_ppc is a power of two >= 8 (cfg_valid).
__device__ __forceinline__ size_t grouped_cell_slot(const Cfg& c, size_t block, int cell, int slot) {
	return (block << c.ppb_shift) + ((slot >> 3) << 9) + (cell << 3) + (slot & 7);
}
// get_block_id (utility_funcs.hpp:21-23): round-half-away-from-zero of p * dx_inv
__device__ __forceinline__ int cell_index(const Cfg& c, float p) { return __float2int_rn(roundf(p * c.dx_inv)); }

// compute_dt (utility_funcs.hpp:36-49) evaluated on the device from the reduced max |v|^2
__device__ __forceinline__ float device_compute_dt(const Cfg& cfg, float max_vel_sq, float step_time, float frame_time, float dt_default) {
	float dt = dt_default;
	const float mv = sqrtf(max_vel_sq);
	if(mv > 0.f) dt = fminf(dt, cfg.dx * cfg.cfl / mv);
	if(frame_time > 0.f) dt = fminf(dt, frame_time - step_time);
	return dt;
}

// A grid node holds mass for the grid update only when its mass is a normal float.  The reference is built with
// --use_fast_math, which flushes subnormal results to zero: a node that only the far corner of a stencil reaches, at
// a weight of order 2^-39 per axis (a particle one ulp from a cell's half below x = 0.5), gets no mass there.  Kept as a
// subnormal, 1 / m overflows to inf, 0 * inf is NaN, and that NaN becomes the particle's velocity and the max |v|^2.
__device__ __forceinline__ bool node_has_mass(float m) { return m >= 1.17549435e-38f; /* FLT_MIN */ }

// max |v|^2 of the two cells a lane holds of a grid block, computed exactly as the grid update will compute it
// (update_grid_velocity_query_max, mgmpm_kernels.cuh:339-388): wall mask, then gravity on y, NaN -> +inf
__device__ __forceinline__ float cell_pair_vel_sq(float2 m, float2 v0, float2 v1, float2 v2, bool wx, bool wy, bool wz, float gdt) {
	float sq0 = 0.f, sq1 = 0.f;
	if(node_has_mass(m.x)) {
		const float mi = 1.f / m.x;
		const float a = wx ? 0.f : v0.x * mi, b = (wy ? 0.f : v1.x * mi) + gdt, c = wz ? 0.f : v2.x * mi;
		sq0 = a * a + b * b + c * c;
	}
	if(node_has_mass(m.y)) {
		const float mi = 1.f / m.y;
		const float a = wx ? 0.f : v0.y * mi, b = (wy ? 0.f : v1.y * mi) + gdt, c = wz ? 0.f : v2.y * mi;
		sq1 = a * a + b * b + c * c;
	}
	if(isnan(sq0)) sq0 = INFINITY;
	if(isnan(sq1)) sq1 = INFINITY;
	return fmaxf(sq0, sq1);
}

// ------------------------------------------------------------------------------------------------
// sm_90a async-proxy primitives (TMA 1-D bulk copy / bulk reduce, mbarrier)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t) __cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, unsigned count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, unsigned bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t* bar, unsigned parity) {
	// the suspend-time hint parks the thread instead of letting 192 of them spin through the issue slots
	asm volatile(
		"{\n"
		".reg .pred p;\n"
		"WAIT_%=:\n"
		"mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n"
		"@p bra DONE_%=;\n"
		"bra WAIT_%=;\n"
		"DONE_%=:\n"
		"}\n" ::"r"(smem_u32(bar)),
		"r"(parity), "r"(0x989680u)
		: "memory");
}
// global -> shared 1-D bulk copy, completion on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, unsigned bytes, uint64_t* bar) {
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// shared -> global 1-D bulk f32 add-reduction performed by the TMA unit at L2 (not an SM-issued atomic)
__device__ __forceinline__ void tma_reduce_add_f32(void* gmem_dst, const void* smem_src, unsigned bytes) {
	asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;" ::"l"(gmem_dst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_store_1d(void* gmem_dst, const void* smem_src, unsigned bytes) {
	asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template<int N>
__device__ __forceinline__ void tma_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template<int N>
__device__ __forceinline__ void tma_wait_all() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
// make generic-proxy smem writes visible to the async proxy before a bulk store/reduce reads them
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// Ampere-style asynchronous 4-byte copy global -> shared (LDGSTS): no destination register, completion by group
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gmem_src) { asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory"); }
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template<int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void prefetch_l1(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// 128-bit streaming global accesses
__device__ __forceinline__ float4 ldg_stream4(const float4* p) {
	float4 r;
	asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
	return r;
}
__device__ __forceinline__ void stg_stream4(float4* p, float4 v) { asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory"); }

}  // namespace cb200
